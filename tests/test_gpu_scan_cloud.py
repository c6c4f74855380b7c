"""Clouds projected from the LaserScans on the device (rpl_scan_cloud_batch_dev, rpl_capsule_stream_scan_cloud_msgs[_dev])
against their definition, oracle/scan_cloud_oracle.py.

The stateless call must be the restatement bit for bit.  Each session case pairs two sessions fed the same pieces, both
with the same filter and footprint tables: every scan-cloud message of one must be P(params, .) of the parsed
laserscan_msgs output of the other, with and without RPL_FLAG_PER_STREAM_FILTERS."""
import math

import numpy as np
import pytest

from oracle import cdr_oracle as CDR
from oracle import scan_cloud_oracle as SC
from test_gpu_scan_filters import CASES, _batch_rows, bits, fleet_filters, flagged
from test_gpu_scan_footprints import FootRowPair, _synth_rows, fleet_footprints
from test_gpu_stream_push_msgs import lidar_settings, pieces_for, receive_times

pytestmark = pytest.mark.gpu

GUARD = 0xA5
CUTOFFS = (-1.0, 0.0, 0.15, 3.0, 7.5, 40.0, 1e9, math.inf)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _cp(R, p):
    return R.scan_cloud_params(p.channels, p.range_cutoff)


# ---- the stateless primitive -------------------------------------------------------------------------------------
def _batch_dev(R, ctx, p, out, time_increment, range_min, range_max):
    import torch

    d = torch.device("cuda", 0)
    n, stride = out["ranges"].shape
    step = SC.point_step(p.channels)
    t = {k: torch.from_numpy(np.ascontiguousarray(out[k])).to(d) for k in ("ranges", "intensities", "angle_increment")}
    tb = torch.from_numpy(np.ascontiguousarray(out["beam_counts"]).view(np.int32)).to(d)
    tt = None if time_increment is None else torch.from_numpy(time_increment).to(d)
    pts = torch.full((n * stride * step + 64,), GUARD, dtype=torch.uint8, device=d)
    cnt = torch.full((n,), -1, dtype=torch.int32, device=d)
    torch.cuda.synchronize()  # the context's stream does not wait for torch's
    ctx.scan_cloud_batch_dev(_cp(R, p), t["ranges"].data_ptr(), t["intensities"].data_ptr(), tb.data_ptr(),
                             t["angle_increment"].data_ptr(), None if tt is None else tt.data_ptr(), range_min,
                             range_max, n, stride, pts.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    return pts.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _check_rows(R, ctx, p, out, ti, lo, hi):
    n, stride = out["ranges"].shape
    step = SC.point_step(p.channels)
    pts, cnt = _batch_dev(R, ctx, p, out, ti, lo, hi)
    want, wcnt = SC.project_rows(p, out["ranges"], out["intensities"], out["beam_counts"], out["angle_increment"], ti,
                                 lo, hi)
    assert cnt.tolist() == wcnt.tolist()
    for s in range(n):
        row = pts[s * stride * step: s * stride * step + int(cnt[s]) * step]
        assert row.tobytes() == want[s].tobytes(), s
    assert (pts[n * stride * step:] == GUARD).all()
    return int(wcnt.sum())


def _with_holes(rng, out):
    """NaN (filtered) and +inf (empty bins) and -inf beams, and ranges on both window edges"""
    out = dict(out)
    r = np.array(out["ranges"], np.float32, copy=True)
    u = rng.random(r.shape)
    r[u < 0.05] = np.nan
    r[(u >= 0.05) & (u < 0.08)] = np.inf
    r[(u >= 0.08) & (u < 0.09)] = -np.inf
    r[(u >= 0.09) & (u < 0.10)] = np.float32(0.15)
    r[(u >= 0.10) & (u < 0.11)] = np.float32(3.0)
    out["ranges"] = r
    return out


@pytest.mark.parametrize("mode_a,inv", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_batch_dev_every_channel_set(R, oracle, mode_a, inv):
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(10 + 2 * mode_a + inv)
    kept = 0
    for ch in range(16):
        base = _batch_rows(R, oracle, ctx, mode_a, inv, 3 * ch + mode_a) if ch % 2 else _synth_rows(rng, mode_a)
        out = _with_holes(rng, base)
        n = out["ranges"].shape[0]
        ti = None if ch % 3 == 0 else rng.uniform(1e-6, 1e-3, n).astype(np.float32)
        cut = CUTOFFS[ch % len(CUTOFFS)]
        kept += _check_rows(R, ctx, SC.params(ch, cut), out, ti, 0.15, 12.0)
    assert kept > 0
    ctx.close()


def test_batch_dev_cutoffs_and_windows(R, oracle):
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(77)
    out = _with_holes(rng, _synth_rows(rng, 1))
    ti = rng.uniform(1e-6, 1e-3, out["ranges"].shape[0]).astype(np.float32)
    for cut in CUTOFFS:
        for lo, hi in ((0.15, 40.0), (0.0, 3.0), (-math.inf, math.inf), (3.0, 3.0)):
            _check_rows(R, ctx, SC.params(SC.CHANNELS, cut), out, ti, lo, hi)
    ctx.close()


def test_batch_dev_refusals(R, oracle):
    import torch

    ctx = R.Context(0, 4096, 4)
    d = torch.device("cuda", 0)
    rows = torch.zeros((4, 4096), dtype=torch.float32, device=d)
    cnt = torch.ones(4, dtype=torch.int32, device=d)
    pts = torch.full((4 * 4096 * 28 + 8,), GUARD, dtype=torch.uint8, device=d)
    a = (rows.data_ptr(), rows.data_ptr(), cnt.data_ptr(), rows.data_ptr(), None, 0.15, 40.0)
    torch.cuda.synchronize()
    bad = R.RESULT_INVALID_DATA
    for p, stride, at in ((R.scan_cloud_params(0x10), 4096, 0), (R.scan_cloud_params(0x13), 4096, 0),
                          (R.scan_cloud_params(range_cutoff=math.nan), 4096, 0), (R.scan_cloud_params(), 4097, 0),
                          (R.scan_cloud_params(), 0, 0), (R.scan_cloud_params(), 4096, 2)):
        with pytest.raises(R.RplError) as e:
            ctx.scan_cloud_batch_dev(p, *a, 4, stride, pts.data_ptr() + at, cnt.data_ptr())
        assert e.value.code == bad
    L = R.lib()
    for k in (1, 2, 3, 4):
        args = list(a[:4])
        args[k - 1] = None
        assert L.rpl_scan_cloud_batch_dev(ctx._h, R.scan_cloud_params(), *args, None, 0.15, 40.0, 4, 4096,
                                          pts.data_ptr(), cnt.data_ptr(), None) == bad
    assert L.rpl_scan_cloud_batch_dev(ctx._h, None, *a, 4, 4096, pts.data_ptr(), cnt.data_ptr(), None) == bad
    assert L.rpl_scan_cloud_batch_dev(ctx._h, R.scan_cloud_params(), *a, 4, 4096, None, cnt.data_ptr(), None) == bad
    assert L.rpl_scan_cloud_batch_dev(ctx._h, R.scan_cloud_params(), *a, 4, 4096, pts.data_ptr(), None, None) == bad
    torch.cuda.synchronize()
    assert (pts.cpu().numpy() == GUARD).all() and (cnt.cpu().numpy() == 1).all()
    ctx.close()


# ---- sessions ----------------------------------------------------------------------------------------------------
PARAMS = [SC.params(SC.DEFAULT), SC.params(SC.CHANNELS, 6.0), SC.params(0), SC.params(SC.TIMESTAMP | SC.DISTANCE, 0.0)]


def projected(msgs, p):
    return [None if m is None else SC.P(p, CDR.parse_laserscan(m)) for m in msgs]


def scan_cloud_dev(R, X, prm, p, off, capacity=None):
    import torch

    ns = X.n_streams * X.max_scans
    per = 288 + 192 + SC.point_step(p.channels) * X.max_nodes + 1
    cap = ns * ((per + 15) // 16 * 16) if capacity is None else capacity
    d = torch.device("cuda", 0)
    store = torch.full((cap + 256,), GUARD, dtype=torch.uint8, device=d)
    offs = torch.full((ns,), -1, dtype=torch.int64, device=d)
    sizes = torch.full((ns,), -1, dtype=torch.int32, device=d)
    total = torch.full((1,), -1, dtype=torch.int64, device=d)
    torch.cuda.synchronize()  # the context's stream does not wait for torch's
    X.scan_cloud_msgs_dev(prm, _cp(R, p), off, store.data_ptr(), cap, offs.data_ptr(), sizes.data_ptr(),
                          total.data_ptr())
    torch.cuda.synchronize()
    return dict(msgs=store.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]), cap=cap)


def check_packed(got, want, cap):
    """exact packing: offsets the exclusive scan of the sizes rounded up to 16, all or nothing, nothing past the end"""
    sizes = [0 if m is None else len(m) for m in want]
    offs = np.concatenate([[0], np.cumsum([(s + 15) // 16 * 16 for s in sizes])[:-1]]).astype(np.uint64)
    total = max([int(o) + s for o, s in zip(offs, sizes) if s] or [0])
    assert got["msg_offsets"].tolist() == offs.tolist()
    assert got["total_bytes"] == total
    fits = total <= cap
    assert got["msg_sizes"].tolist() == [s if fits else 0 for s in sizes]
    buf = got["msgs"]
    if fits:
        for o, m in zip(offs.tolist(), want):
            if m is not None:
                assert bytes(buf[o:o + len(m)]) == m
        assert (buf[total:] == GUARD).all()
    else:
        assert (buf == GUARD).all()
    return total


class CloudPair(FootRowPair):
    """FootRowPair whose A has the same filter and footprint tables as B"""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, fps, lidars=None, types=None):
        super().__init__(R, ctx, kind, ans, n, stride, max_nodes, ms, table, fps, lidars=lidars, types=types)
        self.A.set_scan_filters(self.table)
        self.A.set_scan_footprints(self.fps)
        self.points = self.removed = 0

    def compare_clouds(self, prm, off, dev=False, params=PARAMS):
        R = self.R
        for k, q in enumerate((prm, flagged(R, prm))):
            X, Y = (self.A, self.B) if k else (self.B, self.A)
            scans = Y.laserscan_msgs(q, off)
            for p in params:
                want = projected(scans, p)
                if dev:
                    check_packed(scan_cloud_dev(R, X, q, p, off), want, 1 << 62)
                else:
                    assert X.scan_cloud_msgs(q, _cp(R, p), off) == want
                for w in want:
                    if w is not None:
                        self.points += CDR.parse_pointcloud2(w)["width"]
            if k:  # what the filters and footprints took out of the projection
                plain = projected(Y.laserscan_msgs(prm, off), PARAMS[0])
                got = projected(scans, PARAMS[0])
                self.removed += sum(CDR.parse_pointcloud2(a)["width"] - CDR.parse_pointcloud2(b)["width"]
                                    for a, b in zip(plain, got) if a is not None)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_session_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes; the device cases with per-stream lidar settings mixing Mode A / B and inversion"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 3000)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9700 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    lid = lidar_settings(R, n) if dev else None
    cp = CloudPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n), lidars=lid)
    prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                int(ans % 3 == 0), 1)
    for t, push in enumerate(pieces):
        cp.push(push, prm, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        cp.compare_clouds(prm, 987_654_321 if t % 2 else -5, dev=dev)
    assert cp.points > 0 and cp.removed > 0
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session_with_a_switch(R, oracle, dev):
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x85, 0x86, 0x81, 0x82, 0x83, 0x84]
    n, ms = len(types), 3
    rng = np.random.default_rng(31 + dev)
    before_s = [_streams(oracle, t, 1, 700 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(oracle, t, 1, 800 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    ctx = R.Context(0, 4096, n * ms)
    cp = CloudPair(R, ctx, "bytes", 0, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n), types=types)
    prm = R.scan_params(1, 0, 1, 1)
    for push in p1:
        cp.push(push, prm, dev=dev)
        cp.compare_clouds(prm, 5, dev=dev)
    for x in (cp.A, cp.B):
        x.set_answer_types(after)
    for push in p2:
        cp.push(push, prm, dev=dev)
        cp.compare_clouds(prm, 5, dev=dev)
    assert cp.points > 0
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_several_chunks_disabled_tables_and_emptied_scans(R, oracle, dev):
    """23 streams (device chunks of 7, host chunks of 4); all-disabled filter entries; a stream whose filters remove
    every beam (a width-0 message)"""
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(oracle, 0x82, n, 1900)]
    rng = np.random.default_rng(61 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = (16 << 20) // 5 + 1
    ctx = R.Context(0, 4096, 7 * ms)
    table = [R.scan_filter_settings(enabled=False)] * n
    table[3] = R.scan_filter_settings(range_lo=1e6, range_hi=1e7)  # every beam removed
    cp = CloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, [R.scan_footprint()] * n)
    prm = R.scan_params(0, 1, 0, 1)
    empty = 0
    for push in pieces:
        cp.push(push, prm, dev=dev)
        cp.compare_clouds(prm, 42, dev=dev)
        got = cp.B.scan_cloud_msgs(flagged(R, prm), R.scan_cloud_params(), 42)
        empty += sum(CDR.parse_pointcloud2(m)["width"] == 0 for m in got[3 * ms: 4 * ms] if m is not None)
    assert empty > 0 and cp.points > 0
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """exactly met and one byte short: all or nothing"""
    n, ms = 5, 3
    rng = np.random.default_rng(71 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9900, rng)
    ctx = R.Context(0, 4096, n * ms)
    cp = CloudPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    p = SC.params(SC.CHANNELS)
    tested = 0
    for push in pieces:
        cp.push(push, prm)
        want = projected(cp.A.laserscan_msgs(prm, 3), p)
        full = check_packed(scan_cloud_dev(R, cp.B, prm, p, 3), want, 1 << 62)
        if full == 0:
            continue
        for cap in (full, full - 1):
            if dev:
                check_packed(scan_cloud_dev(R, cp.B, prm, p, 3, capacity=cap), want, cap)
            else:
                store = np.full(cap + 256, GUARD, np.uint8)
                res = cp.B.scan_cloud_msgs(prm, _cp(R, p), 3, msgs=store[:cap], packed=True)
                assert res["result"] == (R.RESULT_OK if cap == full else R.capi.RESULT_INSUFFICIENT_MEMORY)
                assert res["total_bytes"] == full
                if cap == full:
                    res["msgs"] = store
                    check_packed(res, want, cap)
                else:
                    assert (store == GUARD).all()
            tested += 1
    assert tested >= 2
    cp.close()
    ctx.close()


def test_session_refusals(R, oracle):
    import torch

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    bad = R.RESULT_INVALID_DATA
    L = R.lib()
    d = torch.device("cuda", 0)
    store = torch.zeros(1 << 20, dtype=torch.uint8, device=d)
    offs = torch.zeros(n * ms + 1, dtype=torch.int64, device=d)
    sizes = torch.zeros(n * ms + 1, dtype=torch.int32, device=d)
    total = torch.zeros(2, dtype=torch.int64, device=d)
    prm, cp = R.scan_params(1, 0, 0, 1), R.scan_cloud_params()
    a = (store.data_ptr(), 1 << 20, offs.data_ptr(), sizes.data_ptr(), total.data_ptr())
    torch.cuda.synchronize()

    def dev(q, c, *args):
        return L.rpl_capsule_stream_scan_cloud_msgs_dev(fr._h, q, c, 0, *(args or a), None)

    # before any push: nothing to take
    assert dev(prm, cp) == bad
    buf = np.zeros((n, 8, 84), np.uint8)
    fr.push(buf, np.zeros(n, np.uint32), prm)
    assert dev(prm, cp) == R.RESULT_OK
    torch.cuda.synchronize()
    for c in (R.scan_cloud_params(0x10), R.scan_cloud_params(0x20), R.scan_cloud_params(range_cutoff=math.nan)):
        assert dev(prm, c) == bad
        with pytest.raises(R.RplError) as e:
            fr.scan_cloud_msgs(prm, c)
        assert e.value.code == bad
    assert dev(None, cp) == bad and dev(prm, None) == bad
    for k in range(5):
        args = list(a)
        args[k] = None if k != 1 else 1 << 20
        if k != 1:
            assert dev(prm, cp, *args) == bad
    for args in ((store.data_ptr() + 8, *a[1:]), (a[0], a[1], offs.data_ptr() + 4, *a[3:]),
                 (*a[:3], sizes.data_ptr() + 2, a[4]), (*a[:4], total.data_ptr() + 4)):
        assert dev(prm, cp, *args) == bad
    # the flags before set_lidars / set_scan_filters
    for f in (R.FLAG_PER_STREAM, R.FLAG_PER_STREAM_FILTERS):
        assert dev(R.scan_params(1, 0, 0, 1, f), cp) == bad
        with pytest.raises(R.RplError):
            fr.scan_cloud_msgs(R.scan_params(1, 0, 0, 1, f), cp)
    fr.close()
    ctx.close()
