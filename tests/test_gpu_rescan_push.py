"""LaserScans and their re-gridded scans from the push, with a window per stream (rpl_rescan_window_batch_dev,
rpl_capsule_stream_set_rescan_windows, rpl_capsule_stream_push_rescan_msgs[_dev]) against their definition,
oracle/rescan_window_oracle.py.

The stateless call must be W of the restatement bit for bit.  Every session case pairs two sessions fed the same pieces
with the same set calls: A pushes with push_laserscan_msgs and then takes rescan_msgs (the replay, Q without a window),
B takes both from the one call.  B's LaserScan side must be A's push output in every case.  Its re-grid side must be
A's message of every slot whose LaserScan B wrote and whose entry is enabled, packed exactly and written iff it fits,
with the ranges of a stream with a window replaced by W over that stream's qualifying revolutions, which the test keeps
for itself; nothing at or past min(total, capacity) is touched in either buffer."""
import numpy as np
import pytest

from oracle import rescan_oracle as RQ
from oracle import rescan_window_oracle as RW
from test_gpu_rescan import capi_settings, fleet_rescans
from test_gpu_scan_cloud_transforms import XF, XfScanCloudPair, fleet_transforms, frames_for
from test_gpu_scan_filters import fleet_filters, flagged
from test_gpu_scan_footprints import fleet_footprints
from test_gpu_stream_push_msgs import CASES, GUARD, lidar_settings, pieces_for, receive_times
from test_gpu_stream_push_scan_cloud_msgs import exclusive

pytestmark = pytest.mark.gpu

BIG = 288 + 36 + 4 * RQ.MAX_BINS


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


# ---- the stateless call ------------------------------------------------------------------------------------------
def _rows(rng, n, bins):
    a = rng.uniform(0.1, 20.0, (n, bins)).astype(np.float32)
    t = rng.random((n, bins)) < 0.3
    a[t] = np.round(a[t])  # ties
    m = rng.random((n, bins))
    a[m < 0.15] = np.inf
    a[(m >= 0.15) & (m < 0.25)] = np.float32(21.5)  # a seed
    return a


@pytest.mark.parametrize("bins", [1, 7, 360, 4096, 8192])
def test_window_batch_dev_is_the_restatement(R, bins):
    """N 1..16, both statistics, sequences shorter and longer than N"""
    import torch

    ctx = R.Context(0, 4096, 4)
    rng = np.random.default_rng(bins)
    d = torch.device("cuda", 0)
    for n_scans in (3, 21):
        rows = _rows(rng, n_scans, bins)
        tin = torch.from_numpy(rows).to(d)
        for obs in range(1, 17):
            for stat in (RW.MEDIAN, RW.MEAN):
                out = torch.full((n_scans * bins + 8,), -7.0, dtype=torch.float32, device=d)
                torch.cuda.synchronize()
                ctx.rescan_window_batch_dev(R.rescan_window(obs, stat), tin.data_ptr(), n_scans, bins, out.data_ptr())
                torch.cuda.synchronize()
                got = out.cpu().numpy()
                assert (got[n_scans * bins:] == np.float32(-7.0)).all()
                want = RW.window_batch(obs, stat, rows)
                assert (got[: n_scans * bins].view(np.uint32) == want.reshape(-1).view(np.uint32)).all(), (obs, stat)
    ctx.close()


def test_window_batch_dev_refusals(R):
    import ctypes

    import torch

    ctx = R.Context(0, 4096, 4)
    d = torch.device("cuda", 0)
    x = torch.zeros(16, dtype=torch.float32, device=d)
    o = torch.full((16,), -7.0, dtype=torch.float32, device=d)
    torch.cuda.synchronize()
    L = R.lib()
    for obs, stat, bins in ((0, 0, 4), (17, 0, 4), (2, 2, 4), (2, 0, 0), (2, 0, 8193)):
        w = R.RescanWindow(obs, stat)
        assert L.rpl_rescan_window_batch_dev(ctx._h, ctypes.byref(w), x.data_ptr(), 1, bins, o.data_ptr(),
                                             None) == R.RESULT_INVALID_DATA
    w = R.rescan_window(3)
    assert L.rpl_rescan_window_batch_dev(ctx._h, ctypes.byref(w), None, 1, 4, o.data_ptr(), None) == R.RESULT_INVALID_DATA
    assert L.rpl_rescan_window_batch_dev(ctx._h, ctypes.byref(w), x.data_ptr() + 2, 1, 4, o.data_ptr(),
                                         None) == R.RESULT_INVALID_DATA
    torch.cuda.synchronize()
    assert (o.cpu().numpy() == np.float32(-7.0)).all()
    ctx.close()


# ---- sessions ----------------------------------------------------------------------------------------------------
class _Rescanning:
    """B as ScanCloudPair.push_b drives it, with the re-gridding push in place of the projecting one"""

    def __init__(self, B):
        self.B = B

    def push_scan_cloud_msgs(self, *a, cloud_msgs=None, **k):
        return self.B.push_rescan_msgs(*a, rescan_msgs=cloud_msgs, **k)

    def push_scan_cloud_msgs_dev(self, *a, **k):
        return self.B.push_rescan_msgs_dev(*a, **k)


class RescanPushPair(XfScanCloudPair):
    """A: push_laserscan_msgs + rescan_msgs; B: push_rescan_msgs.  The model keeps each stream's window."""

    def __init__(self, R, ctx, *a, **k):
        super().__init__(R, ctx, *a, **k)
        self.ctx = ctx
        self.extra_launches = []  # per push: B's launches beyond A's push_laserscan_msgs on the same input
        self.rescans = []
        self.windows = [(1, RW.MEDIAN)] * self.n
        self.held = [[] for _ in range(self.n)]
        self.windowed = 0

    def _empty(self, mask):
        for s in range(self.n):
            if mask is None or mask[s]:
                self.held[s] = []

    def set_rescans(self, entries, mask=None):
        self.rescans = list(entries) if not self.rescans else [e if mask is None or mask[s] else self.rescans[s]
                                                              for s, e in enumerate(entries)]
        for x in (self.A, self.B):
            x.set_rescans([capi_settings(self.R, e) for e in entries], mask)
        self._empty(mask)

    def set_windows(self, wins, mask=None):
        self.windows = [w if mask is None or mask[s] else self.windows[s] for s, w in enumerate(wins)]
        for x in (self.A, self.B):
            x.set_rescan_windows([self.R.rescan_window(*w) for w in wins], mask)
        self._empty(mask)

    def reset(self, mask):
        self.A.reset(mask)
        self.B.reset(mask)
        self._empty(mask)

    def cloud_big(self, cp):
        return self.n * self.ms * ((BIG + 15) // 16 * 16)

    def push(self, push, prm, cp, off, rx=None, dev=False, scap=None, ccap=None, timing=True):
        buf, cnt = self.buffers(push)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = 64 if (rx is not None and self.kind != "framed") else None
        scap = self.scan_big() if scap is None else scap
        ccap = self.cloud_big(cp) if ccap is None else ccap
        k0 = self.ctx.launch_count
        exp, a_sps = self.A.push_laserscan_msgs(buf, cnt, prm, off, rx_us=rx, timing=tm, chunk_bytes=cb,
                                                msgs=np.zeros(scap, np.uint8), packed=True)
        k1 = self.ctx.launch_count
        a_q = self.A.rescan_msgs(prm, cp, off)
        B = self.B
        self.B = _Rescanning(B)
        k2 = self.ctx.launch_count
        try:
            scans, got = self.push_b(buf, cnt, prm, cp, off, rx, tm, cb, dev, scap, ccap)
        finally:
            self.B = B
        self.extra_launches.append((self.ctx.launch_count - k2) - (k1 - k0))
        assert scans["sps"].tolist() == a_sps.tolist()
        self.check_scans(scans, exp, scap)
        self.check_rescans(got, self.expect(a_q, scans["msg_sizes"]), ccap)
        if scans["result"] is not None:
            over = scans["total_bytes"] > scap or got["total_bytes"] > ccap
            assert scans["result"] == (self.R.capi.RESULT_INSUFFICIENT_MEMORY if over else self.R.RESULT_OK)
        assert a_q == self.A.rescan_msgs(prm, cp, off) == self.B.rescan_msgs(prm, cp, off)  # the replay is Q
        return scans, got

    def expect(self, a_q, scan_sizes):
        """A's message of every slot B wrote a LaserScan for, its ranges windowed; the model's windows advance"""
        want = [None] * len(a_q)
        for s in range(self.n):
            obs, stat = self.windows[s]
            for k in range(self.ms):
                i = s * self.ms + k
                if scan_sizes[i] == 0 or a_q[i] is None:
                    continue
                m = a_q[i]
                if obs == 1:
                    want[i] = m
                    continue
                bins = RQ.ranges_size(self.rescans[s])
                at = len(m) - 4 - 4 * bins
                q = np.frombuffer(m[at: at + 4 * bins], np.float32)
                out, self.held[s] = RW.window_stream(obs, stat, [q], self.held[s])
                want[i] = m[:at] + out[0].tobytes() + m[at + 4 * bins:]
                self.windowed += int(want[i] != m)
        return want

    def check_rescans(self, got, want, cap):
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
            self.n_msgs += 1
        assert (buf[min(total, cap):] == GUARD).all()
        self.cut_clouds += int(total > cap)


def _cps(R):
    return [R.scan_cloud_params(0x03), R.scan_cloud_params(XF | 0x1F, 6.0), R.scan_cloud_params(XF | 0x0C, 0.0)]


def random_windows(rng, n):
    return [(int(rng.integers(1, 17)) if rng.random() < 0.8 else 1, int(rng.integers(0, 2))) for _ in range(n)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_windows_at_one_are_the_replay(R, oracle, kind, ans, dev):
    """every answer type, framed and byte sessions, host and device, stamped and unstamped pushes, filters and
    footprints on every other push, transforms, disabled entries, the windows set to 1 on one pair member's history,
    a reset between pushes; the byte sessions in three chunks of at most three streams, the host and device forms
    alternating on one session"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 7300)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9700 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    chunked = kind == "bytes"
    ctx = R.Context(0, 4096, (3 if chunked else n) * ms)
    p = RescanPushPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                       settings=lidar_settings(R, n) if dev else None)
    p.set_transforms(fleet_transforms(rng, n), frames_for(n))
    p.set_rescans(fleet_rescans(rng, n))
    if ans % 2:
        p.set_windows([(1, int(rng.integers(0, 2))) for _ in range(n)])
    base = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                 int(ans % 3 == 0), 1)
    cps = _cps(R)
    for t, push in enumerate(pieces):
        prm = flagged(R, base) if t % 2 == 0 else base
        form = ((t // 2) % 2 == 0) == dev if chunked else dev
        p.push(push, prm, cps[t % 3], 987_654_321 if t % 2 else -5, rx=rx[t] if t % 2 == 0 else None, dev=form,
               timing=not dev)
        p.compare_after(prm, cps[(t + 1) % 3], 5)
        if t == 1:
            p.reset(np.arange(n) % 2 == 0)
    assert p.n_msgs > n and p.windowed == 0
    if chunked:  # a directory and rescan_kernel per chunk: more than one chunk
        assert max(p.extra_launches) >= 2 * 3
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity_cases(R, oracle, dev):
    """every capacity case of both sets, with and without windows: LaserScans cut (their revolutions skip the window),
    re-grid messages cut (their revolutions still enter it), both, neither"""
    n, ms = 5, 3
    rng = np.random.default_rng(90 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9900, rng)
    ctx = R.Context(0, 4096, n * ms)
    p = RescanPushPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    p.set_transforms(fleet_transforms(rng, n), frames_for(n))
    p.set_rescans(fleet_rescans(rng, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(XF | 0x03)
    for rounds in range(2):
        for t, push in enumerate(pieces):
            scans, got = p.push(push, prm, cp, 3, dev=dev)  # everything fits
            full_s, full_r = scans["total_bytes"], got["total_bytes"]
            if full_s == 0 or full_r == 0:
                continue
            p.reset(None)
            for scap, ccap in ((full_s, full_r - 1), (full_s // 2, None), (full_s - 1, full_r // 3), (full_s, full_r)):
                p.push(push, prm, cp, 3, dev=dev, scap=scap, ccap=ccap)
        p.set_windows(random_windows(rng, n))
    assert p.cut_scans > 0 and p.cut_clouds > 0 and p.windowed > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_random_windows_over_many_pushes(R, oracle, dev):
    """random N and statistic per stream over a dozen pushes and more: pushes that publish nothing, several
    revolutions per stream, masked window and entry updates, and a fleet in seven chunks of three streams, the host and
    device forms alternating on one session"""
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    n, ms = 21, 4
    rng = np.random.default_rng(5 + dev)
    st = [c.reshape(-1) for c in _streams(oracle, 0x84, n, 4400)]
    cuts = [_random_cuts(rng, len(b), [1, 83, 4000, 20000]) for b in st]
    pieces, _ = _pieces_from_cuts(st, cuts)
    # a push that publishes nothing; then the same bytes again, which the sessions take as more of each stream
    pieces = (pieces[:2] + [[np.zeros(0, np.uint8)] * n] + pieces[2:]) * 2
    stride = max(1, max(len(x) for push in pieces for x in push))
    ctx = R.Context(0, 4096, 3 * ms)  # three streams per chunk
    p = RescanPushPair(R, ctx, "bytes", 0x84, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    p.set_transforms(fleet_transforms(rng, n), frames_for(n))
    p.set_rescans(fleet_rescans(rng, n))
    p.set_windows(random_windows(rng, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cps = _cps(R)
    assert len(pieces) >= 12
    for t, push in enumerate(pieces):
        p.push(push, prm, cps[t % 3], 17, dev=(t % 2 == 0) == dev)
        if t % 4 == 3:
            p.set_windows(random_windows(rng, n), (rng.random(n) < 0.3).astype(np.uint8))
        if t % 5 == 4:
            p.set_rescans(fleet_rescans(rng, n), (rng.random(n) < 0.3).astype(np.uint8))
    assert p.windowed > 0 and p.n_msgs > n
    # every chunk has an enabled entry (only every fourth stream is disabled): a directory and rescan_kernel each
    assert min(p.extra_launches) >= 2 * 7
    p.close()
    ctx.close()


def test_state_rules(R, oracle):
    """each emptying event empties exactly the masked streams; refused set calls and refused pushes change nothing;
    a re-layout keeps the unmasked streams' windows"""
    import ctypes

    n, ms = 6, 3
    rng = np.random.default_rng(12)
    streams, pieces, stride = pieces_for(oracle, "bytes", 0x82, n, 9300, rng)
    ctx = R.Context(0, 4096, n * ms)
    p = RescanPushPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    p.set_transforms(fleet_transforms(rng, n), frames_for(n))
    entries = [RQ.settings(-np.pi, np.pi, np.pi / 90, range_max=10.0, use_inf=s % 2 == 0) for s in range(n)]
    p.set_rescans(entries)
    p.set_windows([(1 + 3 * s % 16, s % 2) for s in range(n)])
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(XF | 0x03)
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    for t, push in enumerate(pieces):
        p.push(push, prm, cp, 9, dev=t % 2 == 1)
        mask = (np.arange(n) % 3 == t % 3).astype(np.uint8)
        event = t % 6
        if event == 0:
            p.reset(mask)
        elif event == 1:
            p.set_windows([(int(rng.integers(2, 17)), int(rng.integers(0, 2))) for _ in range(n)], mask)
        elif event == 2:
            p.set_rescans(fleet_rescans(rng, n), mask)
        elif event == 3:  # export and import into the same streams: the carried state is unchanged, the window not
            idx = np.flatnonzero(mask)
            for x in (p.A, p.B):
                rec, off = x.export_streams(idx)
                x.import_streams(idx, rec, off)
            p._empty(mask)
        elif event == 4:  # refused set calls and a refused push leave every window as it was
            wins = (R.RescanWindow * n)(*[R.rescan_window(17)] * n)
            assert L.rpl_capsule_stream_set_rescan_windows(p.B._h, ctypes.cast(wins, ctypes.c_void_p), None) == bad
            assert L.rpl_capsule_stream_set_rescan_windows(p.B._h, None, None) == bad
            ents = (R.capi.RescanSettings * n)(*[R.rescan_settings(angle_increment=0.0)] * n)
            assert L.rpl_capsule_stream_set_rescans(p.B._h, ctypes.cast(ents, ctypes.c_void_p), None) == bad
            with pytest.raises(R.RplError):
                p.B.push_rescan_msgs(np.zeros((n, stride), np.uint8), np.zeros(n, np.uint32), prm,
                                     R.scan_cloud_params(0x10), 9)
        elif event == 5:  # a re-layout from the other table: the masked streams empty, the others keep theirs
            p.set_rescans([RQ.settings(-1.0, 1.0, 0.004, range_max=8.0)] * n, mask)
    assert p.windowed > 0
    p.close()
    ctx.close()


def test_answer_type_switch_empties_the_switched_streams(R, oracle):
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x81, 0x86, 0x83, 0x82, 0x85, 0x84]  # streams 1, 3, 5 switch
    n, ms = len(types), 3
    rng = np.random.default_rng(66)
    b1 = [_streams(oracle, t, 1, 930 + s)[0].reshape(-1) for s, t in enumerate(types)]
    b2 = [_streams(oracle, t, 1, 940 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(b1, [cut(b) for b in b1])
    p2, _ = _pieces_from_cuts(b2, [cut(b) for b in b2])
    stride = max(len(x) for push in p1 + p2 for x in push)
    ctx = R.Context(0, 4096, n * ms)
    p = RescanPushPair(R, ctx, "bytes", 0, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                       types=types)
    p.set_rescans([RQ.settings(range_max=12.0)] * n)
    p.set_windows([(5, RW.MEDIAN), (3, RW.MEAN)] * 3)
    prm = flagged(R, R.scan_params(1, 0, 1, 1))
    cp = R.scan_cloud_params(0x03)
    for push in p1:
        p.push(push, prm, cp, 5)
    for x in (p.A, p.B):
        x.set_answer_types(after)
    p._empty(np.array(types) != np.array(after))
    for t, push in enumerate(p2):
        p.push(push, prm, cp, 5, dev=t % 2 == 1)
    assert p.windowed > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("per_chunk", [5, 2])
def test_launch_counts(R, oracle, per_chunk):
    """the existing calls launch what they launched before any window; a chunk with no enabled entry launches no
    re-grid kernel, and one with no window no window kernel; one chunk, or three of at most two streams"""
    n, ms = 5, 3
    rng = np.random.default_rng(31)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9600, rng)
    ctx = R.Context(0, 4096, per_chunk * ms)
    p = RescanPushPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(0x03)
    B = p.B
    buf, cnt = p.buffers(pieces[0])

    def count(fn):
        k = ctx.launch_count
        fn()
        return ctx.launch_count - k

    laser = lambda: B.push_laserscan_msgs(buf, cnt, prm, 0, packed=True)  # noqa: E731
    clouds = lambda: B.push_scan_cloud_msgs(buf, cnt, prm, cp, 0)  # noqa: E731
    rescan = lambda: B.push_rescan_msgs(buf, cnt, prm, cp, 0)  # noqa: E731
    replay = lambda: B.rescan_msgs(prm, cp, 0)  # noqa: E731
    base_l, base_c = count(laser), count(clouds)
    p.set_rescans([RQ.settings(enabled=False)] * n)
    base_r = count(replay)
    dirs = count(rescan) - base_l  # one re-grid directory per chunk, and nothing else
    assert dirs == -(-n // per_chunk)
    p.set_rescans([RQ.settings()] * n)
    assert count(rescan) == base_l + 2 * dirs  # and rescan_kernel per chunk
    p.set_windows([(1, 0)] * n)
    assert count(rescan) == base_l + 2 * dirs
    assert (count(laser), count(clouds)) == (base_l, base_c)
    p.set_windows([(4, 1)] + [(1, 0)] * (n - 1))
    assert count(rescan) == base_l + 2 * dirs + 1  # and the window kernel in the first chunk
    p.set_windows([(4, 1)] + [(1, 0)] * (n - 2) + [(3, 0)])
    assert count(rescan) == base_l + 2 * dirs + (1 if dirs == 1 else 2)  # the first and the last chunk's
    assert (count(laser), count(clouds)) == (base_l, base_c)
    p.set_rescans([RQ.settings(enabled=False)] * n)
    assert count(replay) == base_r
    p.close()
    ctx.close()
