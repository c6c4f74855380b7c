"""Merged scans from the push (rpl_rescan_merge_batch_dev, rpl_capsule_stream_set_rescan_merges,
rpl_capsule_stream_push_rescan_merge_msgs[_dev]) against their definition, oracle/rescan_merge_oracle.py.

The stateless call must be M of the restatement bit for bit.  Every session case pairs two sessions fed the same pieces
with the same set calls, as test_gpu_rescan_push.py does: A pushes with push_laserscan_msgs and takes the rescan_msgs
replay, B takes everything from the merge call.  B's LaserScans and re-grid messages must be what that file's pair
checks for push_rescan_msgs (A's messages, windowed), and B's merged messages must be the session model of the oracle
fed the re-grid messages B wrote, packed by group, with nothing touched at or past min(total, capacity)."""
import ctypes

import numpy as np
import pytest

from oracle import rescan_merge_oracle as RM
from oracle import rescan_oracle as RQ
from oracle import rescan_window_oracle as RW
from test_gpu_rescan import GRIDS, capi_settings
from test_gpu_rescan_push import RescanPushPair, _cps
from test_gpu_scan_cloud_transforms import XF, random_entry
from test_gpu_scan_filters import fleet_filters, flagged
from test_gpu_scan_footprints import fleet_footprints
from test_gpu_stream_push_msgs import CASES, GUARD, lidar_settings, pieces_for, receive_times
from test_gpu_stream_push_scan_cloud_msgs import fleet

pytestmark = pytest.mark.gpu

BIG = 288 + 36 + 4 * RQ.MAX_BINS
NONE = RM.NONE


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


# ---- the stateless call ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", range(5))
def test_merge_batch_dev_is_the_restatement(R, g):
    """bins 1, 7, 360, 4096, 8192; groups of 0, 1, 2, 4 and many rows, rows of no group, both seeds, guard words"""
    import torch

    ctx = R.Context(0, 4096, 4)
    rng = np.random.default_rng(70 + g)
    d = torch.device("cuda", 0)
    for use_inf in (True, False):
        s = RQ.settings(*GRIDS[g], range_max=11.0, use_inf=use_inf, inf_epsilon=0.5)
        bins = RQ.ranges_size(s)
        assert bins == [1, 7, 360, 4096, 8192][g]
        n_groups = 6
        row_group = [0, 1, 1, NONE] + [2] * 4 + [4] * 19 + [NONE, 7]  # groups 3 and 5 empty, 7 past n_groups
        rows = rng.uniform(0.1, 12.0, (len(row_group), bins)).astype(np.float32)
        rows[rng.random(rows.shape) < 0.2] = np.inf
        rows[rng.random(rows.shape) < 0.1] = RQ.seed(s)
        tin = torch.from_numpy(rows).to(d)
        tg = torch.from_numpy(np.array(row_group, np.uint32).view(np.int32)).to(d)
        out = torch.full((n_groups * bins + 8,), -7.0, dtype=torch.float32, device=d)
        torch.cuda.synchronize()
        ctx.rescan_merge_batch_dev(capi_settings(R, s), tin.data_ptr(), tg.data_ptr(), len(row_group), n_groups,
                                   out.data_ptr())
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert (got[n_groups * bins:] == np.float32(-7.0)).all()
        want = RM.merge_batch(s, rows, row_group, n_groups)
        assert (got[: n_groups * bins].view(np.uint32) == want.reshape(-1).view(np.uint32)).all(), use_inf
    ctx.close()


def test_merge_batch_dev_refusals(R):
    import torch

    ctx = R.Context(0, 4096, 4)
    d = torch.device("cuda", 0)
    x = torch.zeros(16, dtype=torch.float32, device=d)
    gi = torch.zeros(4, dtype=torch.int32, device=d)
    o = torch.full((16,), -7.0, dtype=torch.float32, device=d)
    torch.cuda.synchronize()
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    ok = R.rescan_settings(0.0, 1.0, 0.25)
    for s in (R.rescan_settings(angle_increment=0.0), R.rescan_settings(0.0, 1.0, 1e-5)):
        assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(s), x.data_ptr(), gi.data_ptr(), 2, 2, o.data_ptr(),
                                            None) == bad
    assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(ok), None, gi.data_ptr(), 2, 2, o.data_ptr(), None) == bad
    assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(ok), x.data_ptr(), None, 2, 2, o.data_ptr(), None) == bad
    assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(ok), x.data_ptr(), gi.data_ptr(), 2, 2, None, None) == bad
    assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(ok), x.data_ptr() + 2, gi.data_ptr(), 2, 2, o.data_ptr(),
                                        None) == bad
    assert L.rpl_rescan_merge_batch_dev(ctx._h, ctypes.byref(ok), x.data_ptr(), gi.data_ptr(), 2, 2, o.data_ptr() + 1,
                                        None) == bad
    torch.cuda.synchronize()
    assert (o.cpu().numpy() == np.float32(-7.0)).all()
    ctx.close()


# ---- sessions ----------------------------------------------------------------------------------------------------
class _Merging:
    """B as RescanPushPair drives it, with the merge push in place of push_rescan_msgs; the merged set goes to the
    pair"""

    def __init__(self, B, pair):
        self.B, self.pair = B, pair

    def push_scan_cloud_msgs(self, *a, cloud_msgs=None, **k):
        p = self.pair
        store = np.full(p.mcap_now + 256, GUARD, np.uint8)
        scans, rescans, merged, sps = self.B.push_rescan_merge_msgs(*a[:4], p.n_groups, *a[4:], rescan_msgs=cloud_msgs,
                                                                    merged_msgs=store[:p.mcap_now], **k)
        merged["msgs"] = store
        p.merged_out, p.rc = merged, scans["result"]
        scans["result"] = rescans["result"] = None  # checked against all three totals by MergePair
        return scans, rescans, sps

    def push_scan_cloud_msgs_dev(self, *a, **k):
        import torch

        p = self.pair
        d = torch.device("cuda", 0)
        G = max(p.n_groups, 1)
        t = dict(store=torch.full((p.mcap_now + 256,), GUARD, dtype=torch.uint8, device=d),
                 offs=torch.full((G,), -1, dtype=torch.int64, device=d),
                 sizes=torch.full((G,), -1, dtype=torch.int32, device=d),
                 total=torch.full((1,), -1, dtype=torch.int64, device=d))
        out = p.R.MsgsOut(t["store"].data_ptr(), p.mcap_now, t["offs"].data_ptr(), t["sizes"].data_ptr(),
                          t["total"].data_ptr())
        p.merged_dev, p.rc = t, None
        torch.cuda.synchronize()
        return self.B.push_rescan_merge_msgs_dev(*a[:7], out, *a[7:], **k)


class MergePair(RescanPushPair):
    """RescanPushPair whose B takes the merge push; the oracle's session model keeps the held grids"""

    def __init__(self, R, ctx, *a, **k):
        super().__init__(R, ctx, *a, **k)
        self.model = RM.MergeModel(self.n)
        self.n_groups = 0
        self.mcap_now = 0
        self.merged_msgs = 0
        self.stale = 0  # merged messages with a contributor from an earlier push

    def _empty(self, mask):
        super()._empty(mask)
        self.model.empty(mask)

    def set_merges(self, group_of_stream, max_age):
        assert self.model.set_merges(group_of_stream, max_age)
        self.B.set_rescan_merges(group_of_stream, max_age)
        self.n_groups = len(max_age)

    def set_transforms(self, entries, frames, mask=None):
        super().set_transforms(entries, frames, mask)
        self.model.empty(mask)

    def push_b(self, *a):
        inner = self.B
        self.B = _Merging(inner.B, self)
        try:
            return super().push_b(*a)
        finally:
            self.B = inner

    def push(self, push, prm, cp, off, rx=None, dev=False, scap=None, ccap=None, mcap=None, timing=True):
        self.mcap_now = max(self.n_groups, 1) * ((BIG + 15) // 16 * 16) if mcap is None else mcap
        self.merged_out = self.merged_dev = None
        scans, got = super().push(push, prm, cp, off, rx=rx, dev=dev, scap=scap, ccap=ccap, timing=timing)
        if self.merged_dev is not None:
            t = self.merged_dev
            G = self.n_groups
            self.merged_out = dict(msgs=t["store"].cpu().numpy(),
                                   msg_offsets=t["offs"].cpu().numpy()[:G].view(np.uint64),
                                   msg_sizes=t["sizes"].cpu().numpy()[:G].view(np.uint32),
                                   total_bytes=int(t["total"].cpu().numpy()[0]))
        written = [[] for _ in range(self.n)]
        for s in range(self.n):
            for k in range(self.ms):
                i = s * self.ms + k
                n = int(got["msg_sizes"][i])
                if n:
                    o = int(got["msg_offsets"][i])
                    written[s].append(bytes(got["msgs"][o:o + n]))
        m = self.model
        want = m.push(written, lambda s: self.rescans[s])
        self.check_merged(self.merged_out, want)
        self.stale += sum(1 for g, w in enumerate(want) if w is not None and any(
            m.held[s] is not None and 0 < m.seq - m.held[s][1] <= m.max_age[g] for s in m.groups[g]))
        if self.rc is not None:
            over = (scans["total_bytes"] > (self.scan_big() if scap is None else scap) or
                    got["total_bytes"] > (self.cloud_big(cp) if ccap is None else ccap) or
                    self.merged_out["total_bytes"] > self.mcap_now)
            assert self.rc == (self.R.capi.RESULT_INSUFFICIENT_MEMORY if over else self.R.RESULT_OK)
        return scans, got, self.merged_out

    def check_merged(self, got, want):
        offs, sizes, total = RM.pack(want, self.mcap_now)
        assert got["msg_offsets"].tolist() == offs
        assert got["msg_sizes"].tolist() == sizes
        assert got["total_bytes"] == total
        buf = got["msgs"]
        for g, n in enumerate(sizes):
            if n:
                assert bytes(buf[offs[g]:offs[g] + n]) == want[g], g
                self.merged_msgs += 1
        assert (buf[min(total, self.mcap_now):] == GUARD).all()


def grouped(rng, n, n_groups, every=3):
    """every `every`-th stream in no group, the others spread over n_groups groups (each at least one member)"""
    g = [NONE if s % every == every - 1 else 0 for s in range(n)]
    members = [s for s in range(n) if g[s] != NONE]
    for j, s in enumerate(members):
        g[s] = j % n_groups if j < n_groups else int(rng.integers(0, n_groups))
    return g


def group_tables(rng, R, groups, n):
    """one re-grid entry, LaserScan frame and target frame per group; transforms all enabled"""
    ents, frames, targets = [], [], []
    gs = sorted({x for x in groups if x != NONE})
    ge = {g: RQ.settings(*GRIDS[(g + 2) % len(GRIDS)], range_max=float(rng.uniform(5, 12)), min_height=-0.3,
                         max_height=0.6, use_inf=g % 2 == 0, inf_epsilon=0.5) for g in gs}
    for s in range(n):
        g = groups[s]
        ents.append(ge[g] if g != NONE else RQ.settings(*GRIDS[s % len(GRIDS)], enabled=s % 4 != 3))
        frames.append("laser_g%d" % g if g != NONE else "laser_%d" % s)
        targets.append("base_link" if g != NONE and g % 2 == 0 else ("base_g%d" % g if g != NONE else "t%d" % s))
    return ents, frames, targets


def setup_pair(R, ctx, rng, kind, ans, n, stride, ms, groups, max_age, settings=None, types=None, windows=None):
    ents, frames, targets = group_tables(rng, R, groups, n)
    p = MergePair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                  settings=settings, types=types)
    for x in (p.A, p.B):
        x.set_frames(frames)
    p.frames = frames
    p.set_transforms([random_entry(rng, True) for _ in range(n)], targets)
    p.set_rescans(ents)
    if windows:
        p.set_windows(windows)
    p.set_merges(groups, max_age)
    return p


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_merged_scans_are_the_model(R, oracle, kind, ans, dev):
    """every answer type, framed and byte sessions, host and device, stamped and unstamped pushes, filters and
    footprints, 3-D transforms with and without the bit (the LaserScan frames are grouped too), a reset between pushes,
    a group of one; the byte sessions in chunks of three streams"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 8100)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9700 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    chunked = kind == "bytes"
    ctx = R.Context(0, 4096, (3 if chunked else n) * ms)
    groups = [0, 1, 0, NONE, 1, 2, 1]  # group 2 has one member
    p = setup_pair(R, ctx, rng, kind, ans, n, stride, ms, groups, [0, 3, 1],
                   settings=lidar_settings(R, n) if dev else None)
    base = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                 int(ans % 3 == 0), 1)
    cps = _cps(R)
    for t, push in enumerate(pieces):
        prm = flagged(R, base) if t % 2 == 0 else base
        p.push(push, prm, cps[t % 3], 987_654_321 if t % 2 else -5, rx=rx[t] if t % 2 == 0 else None, dev=dev,
               timing=not dev)
        if t == 1:
            p.reset(np.arange(n) % 2 == 0)
    assert p.merged_msgs > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_fleet_groups_across_chunks_with_windows_and_ages(R, oracle, dev):
    """23 streams (device chunks of 3, host chunks of 4), groups whose members span chunks, ungrouped streams, median
    and mean windows next to unwindowed members, max_age 0 and 3 with streams idle for whole pushes"""
    n, ms, pieces, stride, rx, table = fleet(R, oracle, 1700)
    rng = np.random.default_rng(1700 + dev)
    ctx = R.Context(0, 4096, 3 * ms)
    groups = grouped(rng, n, 4)
    wins = [(int(rng.integers(2, 8)), int(rng.integers(0, 2))) if s % 2 else (1, 0) for s in range(n)]
    p = setup_pair(R, ctx, rng, "bytes", 0x82, n, stride, ms, groups, [0, 3, 3, 1], windows=wins)
    prm = flagged(R, R.scan_params(0, 1, 0, 1))
    cps = _cps(R)
    for rnd in range(2):
        for t, push in enumerate(pieces):
            idle = rng.random(n) < 0.3  # whole pushes without a byte for these streams
            push = [np.zeros(0, np.uint8) if idle[s] else x for s, x in enumerate(push)]
            p.push(push, prm, cps[(t + rnd) % 3], 42, dev=(t % 2 == 0) == dev)
    assert p.merged_msgs > n and p.stale > 0 and p.windowed > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity_cases(R, oracle, dev):
    """all three capacities exactly met and one byte short, each alone, with guard bytes"""
    n, ms = 6, 3
    rng = np.random.default_rng(190 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9900, rng)
    ctx = R.Context(0, 4096, n * ms)
    p = setup_pair(R, ctx, rng, "framed", 0x85, n, stride, ms, [0, 1, 2, 0, 1, 2], [2, 2, 2])
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(XF | 0x03)
    cut = 0
    for t, push in enumerate(pieces):
        scans, got, merged = p.push(push, prm, cp, 3, dev=dev)
        fs, fr, fm = scans["total_bytes"], got["total_bytes"], merged["total_bytes"]
        if not (fs and fr and fm):
            continue
        for caps in ((fs, fr, fm), (fs - 1, fr, fm), (fs, fr - 1, fm), (fs, fr, fm - 1), (fs, fr, fm // 2)):
            p.reset(None)
            p.push(push, prm, cp, 3, dev=dev, scap=caps[0], ccap=caps[1], mcap=caps[2])
            cut += 1
    assert cut > 0 and p.cut_scans > 0 and p.cut_clouds > 0
    p.close()
    ctx.close()


def test_emptying_rules_and_refusals(R, oracle):
    """each emptying call empties exactly the masked streams' held grids; every refusal leaves seq, held grids and
    windows as they were"""
    n, ms = 6, 3
    rng = np.random.default_rng(12)
    streams, pieces, stride = pieces_for(oracle, "bytes", 0x82, n, 9300, rng)
    ctx = R.Context(0, 4096, n * ms)
    groups = [0, 0, 1, 1, 1, NONE]
    p = setup_pair(R, ctx, rng, "bytes", 0x82, n, stride, ms, groups, [5, 5], windows=[(3, 0)] * n)
    ents, frames, targets = list(p.rescans), p.frames, group_tables(rng, R, groups, n)[2]
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(XF | 0x03)
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    B = p.B
    def refused_push(cpx=cp, merged=True, dev_off=0):
        import torch

        d = torch.device("cuda", 0)
        ns = n * ms
        bufs = [torch.zeros(1 << 20, dtype=torch.uint8, device=d) for _ in range(3)]
        tabs = [(torch.zeros(ns, dtype=torch.int64, device=d), torch.zeros(ns, dtype=torch.int32, device=d),
                 torch.zeros(1, dtype=torch.int64, device=d)) for _ in range(3)]
        outs = [R.MsgsOut(b.data_ptr() + (dev_off if k == 2 else 0), 1 << 19, o.data_ptr(), z.data_ptr(), t.data_ptr())
                for k, (b, (o, z, t)) in enumerate(zip(bufs, tabs))]
        data = torch.zeros((n, stride), dtype=torch.uint8, device=d)
        cnt = torch.zeros(n, dtype=torch.int32, device=d)
        sps = torch.zeros(n, dtype=torch.int32, device=d)
        pi = B._push_input(data.data_ptr(), cnt.data_ptr(), 31, None, None, None)
        torch.cuda.synchronize()
        rc = L.rpl_capsule_stream_push_rescan_merge_msgs_dev(B._h, ctypes.byref(pi), ctypes.byref(prm),
                                                             ctypes.byref(cpx), 0, ctypes.byref(outs[0]),
                                                             ctypes.byref(outs[1]),
                                                             ctypes.byref(outs[2]) if merged else None,
                                                             sps.data_ptr(), None)
        torch.cuda.synchronize()
        assert rc == bad

    for t, push in enumerate(pieces):
        p.push(push, prm, cp, 9, dev=t % 2 == 1)
        mask = (np.arange(n) % 3 == t % 3).astype(np.uint8)
        event = t % 9
        if event == 0:
            p.reset(mask)
        elif event == 1:
            p.set_windows([(int(rng.integers(1, 6)), int(rng.integers(0, 2))) for _ in range(n)], mask)
        elif event == 2:
            p.set_rescans(ents, mask)
        elif event == 3:  # export and import into the same streams: the held grids do not travel
            idx = np.flatnonzero(mask)
            for x in (p.A, p.B):
                rec, off = x.export_streams(idx)
                x.import_streams(idx, rec, off)
            p._empty(mask)
        elif event == 4:
            p.set_transforms([random_entry(rng, True) for _ in range(n)], targets, mask)
        elif event == 5:  # set_frames empties every stream
            for x in (p.A, p.B):
                x.set_frames(frames)
            p._empty(None)
        elif event == 6:  # refused set calls
            gs = (ctypes.c_uint32 * n)(*[0, 0, 2, 1, 1, NONE])  # index 2 with two groups
            ages = (ctypes.c_uint32 * 2)(1, 1)
            assert L.rpl_capsule_stream_set_rescan_merges(B._h, gs, ages, 2) == bad
            gs = (ctypes.c_uint32 * n)(*[0, 0, 0, 0, 0, NONE])  # group 1 is empty
            assert L.rpl_capsule_stream_set_rescan_merges(B._h, gs, ages, 2) == bad
            assert L.rpl_capsule_stream_set_rescan_merges(B._h, gs, (ctypes.c_uint32 * 1)(65536), 1) == bad
            assert L.rpl_capsule_stream_set_rescan_merges(B._h, gs, (ctypes.c_uint32 * 7)(*[0] * 7), 7) == bad
        elif event == 7:  # refused pushes: null merged, misaligned merged, frames that differ without the bit
            refused_push(merged=False)
            refused_push(dev_off=8)
        elif event == 8:  # mismatched and disabled entries: refused until they agree again
            e2 = list(ents)
            e2[1] = RQ.settings(*GRIDS[3])
            p.set_rescans(e2, np.eye(n, dtype=np.uint8)[1])
            refused_push()
            e2[1] = RQ.settings(**{**vars(ents[0]), "enabled": False})
            p.set_rescans(e2, np.eye(n, dtype=np.uint8)[1])
            refused_push()
            p.set_rescans(ents, np.eye(n, dtype=np.uint8)[1])
    assert p.merged_msgs > 0 and p.stale > 0
    p.close()
    ctx.close()


def test_frames_are_checked_per_call_and_refusals_change_nothing(R, oracle):
    """LaserScan frames that differ within a group: a push with the transform bit merges (one target frame), one
    without it is refused and leaves seq and held grids as they were; a push before set_rescan_merges is refused"""
    n, ms = 4, 3
    rng = np.random.default_rng(44)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x84, n, 9400, rng)
    ctx = R.Context(0, 4096, n * ms)
    groups = [0, 0, 1, 1]
    ents, frames, targets = group_tables(rng, R, groups, n)
    p = MergePair(R, ctx, "framed", 0x84, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    for x in (p.A, p.B):
        x.set_frames(["a", "b", "c", "d"])  # every stream's own LaserScan frame
    p.frames = ["a", "b", "c", "d"]
    p.set_transforms([random_entry(rng, True) for _ in range(n)], targets)
    p.set_rescans(ents)
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    with pytest.raises(R.RplError):  # before set_rescan_merges
        p.B.push_rescan_merge_msgs(np.zeros((n, stride, p.B.capsule_bytes), np.uint8), np.zeros(n, np.uint32), prm,
                                   R.scan_cloud_params(XF | 0x03), 0)
    p.set_merges(groups, [4, 4])
    for t, push in enumerate(pieces):
        p.push(push, prm, R.scan_cloud_params(XF | 0x03), 5, dev=t % 2 == 0)
        with pytest.raises(R.RplError):
            p.B.push_rescan_merge_msgs(np.zeros((n, stride, p.B.capsule_bytes), np.uint8), np.zeros(n, np.uint32),
                                       prm, R.scan_cloud_params(0x03), 2)
    assert p.merged_msgs > 0
    p.close()
    ctx.close()


def test_answer_type_switch_empties_the_switched_streams(R, oracle):
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x81, 0x86, 0x83, 0x82, 0x85, 0x84]  # streams 1, 3, 5 switch
    n, ms = len(types), 3
    rng = np.random.default_rng(67)
    b1 = [_streams(oracle, t, 1, 930 + s)[0].reshape(-1) for s, t in enumerate(types)]
    b2 = [_streams(oracle, t, 1, 940 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(b1, [cut(b) for b in b1])
    p2, _ = _pieces_from_cuts(b2, [cut(b) for b in b2])
    stride = max(len(x) for push in p1 + p2 for x in push)
    ctx = R.Context(0, 4096, n * ms)
    p = setup_pair(R, ctx, rng, "bytes", 0, n, stride, ms, [0, 0, 0, 1, 1, 1], [9, 9], types=types,
                   windows=[(5, RW.MEDIAN), (1, 0)] * 3)
    prm = flagged(R, R.scan_params(1, 0, 1, 1))
    cp = R.scan_cloud_params(XF | 0x03)
    for push in p1:
        p.push(push, prm, cp, 5)
    for x in (p.A, p.B):
        x.set_answer_types(after)
    p._empty(np.array(types) != np.array(after))
    for t, push in enumerate(p2):
        p.push(push, prm, cp, 5, dev=t % 2 == 1)
    assert p.merged_msgs > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("per_chunk", [5, 2])
def test_launch_counts(R, oracle, per_chunk):
    """a chunk without a grouped stream makes no hold launch; the end adds the directory and the merge kernel; the
    existing calls launch what they launched before any group"""
    n, ms = 5, 3
    rng = np.random.default_rng(31)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9600, rng)
    ctx = R.Context(0, 4096, per_chunk * ms)
    p = MergePair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp = R.scan_cloud_params(0x03)
    B = p.B
    buf, cnt = p.buffers(pieces[0])

    def count(fn):
        k = ctx.launch_count
        fn()
        return ctx.launch_count - k

    p.set_rescans([RQ.settings()] * n)
    for x in (p.A, B):
        x.set_frames(["laser"] * n)
    p.frames = ["laser"] * n
    laser = lambda: B.push_laserscan_msgs(buf, cnt, prm, 0, packed=True)  # noqa: E731
    clouds = lambda: B.push_scan_cloud_msgs(buf, cnt, prm, cp, 0)  # noqa: E731
    rescan = lambda: B.push_rescan_msgs(buf, cnt, prm, cp, 0)  # noqa: E731
    before = (count(laser), count(clouds), count(rescan))
    chunks = -(-n // per_chunk)
    B.set_rescan_merges([NONE] * n, [])
    assert count(lambda: B.push_rescan_merge_msgs(buf, cnt, prm, cp, 0, 0)) == before[2] + 1  # the directory alone
    B.set_rescan_merges([NONE] * (n - 1) + [0], [1])  # the last chunk only
    assert count(lambda: B.push_rescan_merge_msgs(buf, cnt, prm, cp, 0, 1)) == before[2] + 1 + 2
    B.set_rescan_merges([0] + [NONE] * (n - 2) + [0], [1])  # the first and the last chunk
    assert count(lambda: B.push_rescan_merge_msgs(buf, cnt, prm, cp, 0, 1)) == before[2] + min(chunks, 2) + 2
    assert (count(laser), count(clouds), count(rescan)) == before
    p.close()
    ctx.close()
