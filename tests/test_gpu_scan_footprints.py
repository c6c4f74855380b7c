"""The footprint stage of the LaserScan filters on the device (rpl_scan_filter_footprint_batch_dev,
rpl_capsule_stream_set_scan_footprints) against its definition, oracle/scan_footprint_oracle.py.

The stateless call must be the restatement bit for bit.  The session cases pair two sessions fed the same pieces, as
tests/test_gpu_scan_filters.py does: A makes the call without RPL_FLAG_PER_STREAM_FILTERS and the restatement F(filter
entry s, footprint s, scan) is applied to its outputs on the host, B has the footprints and makes the flagged call."""
import math

import numpy as np
import pytest

from oracle import scan_footprint_oracle as FP
from test_gpu_scan_filters import CASES, STAGES, MsgPair, RowPair, _batch_rows, bits, fleet_filters, flagged
from test_gpu_stream_push_msgs import CHUNK, Pair, lidar_settings, pieces_for, receive_times
from test_scan_footprints_oracle import BAD, GOOD, _star, make

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def fleet_footprints(R, n):
    """a body with the lidar at a corner, a box, a region of interest, four 16-vertex polygons, an L-shape, none"""
    rng = np.random.default_rng(7)
    table = [
        R.scan_footprint([[(-1.5, -1.0), (1.5, -1.0), (1.5, 1.0), (-1.5, 1.0)]], pose=(1.5, 1.0, math.radians(45))),
        R.scan_footprint([[(-2.0, -1.0), (2.0, -1.0), (2.0, 1.0), (-2.0, 1.0)]]),
        R.scan_footprint([[(-1.0, -4.0), (6.0, 0.0), (-1.0, 4.0)]], invert=[1], pose=(-0.5, 0.2, 0.3)),
        R.scan_footprint([_star(rng, 16, *rng.uniform(-2, 2, 2), 0.5, 5.0) for _ in range(4)], invert=[0, 1, 0, 0],
                         pose=(0.3, -0.4, 2.0)),
        R.scan_footprint([[(0.0, 0.0), (4.0, 0.0), (4.0, 2.0), (2.0, 2.0), (2.0, 4.0), (0.0, 4.0)]],
                         pose=(1.0, 1.0, -2.5)),
        R.scan_footprint(),
    ]
    return [table[s % len(table)] for s in range(n)]


def random_footprint(R, rng):
    k = int(rng.integers(1, 5))
    return R.scan_footprint([_star(rng, int(rng.integers(3, 17)), *rng.uniform(-3, 3, 2), 0.2, 8.0) for _ in range(k)],
                            invert=[int(rng.random() < 0.3) for _ in range(k)],
                            pose=(*rng.uniform(-2, 2, 2), rng.uniform(-7, 7)))


def filter_msg(m, e, fp):
    """F(e, fp, .) applied to one serialised LaserScan: the ranges rewritten in place, everything else as it is"""
    if m is None:
        return None
    L = int(np.frombuffer(m, "<u4", 1, 12)[0])  # frame_id length with its NUL
    hb = 4 + ((12 + L + 3) & ~3)
    inc = np.frombuffer(m, "<f4", 1, hb + 8)[0]
    M = int(np.frombuffer(m, "<u4", 1, hb + 28)[0])
    r = np.frombuffer(m, "<f4", M, hb + 32)
    it = np.frombuffer(m, "<f4", M, hb + 32 + 4 * M + 4)
    return m[:hb + 32] + FP.filter_scan(e, fp, r, it, inc).tobytes() + m[hb + 32 + 4 * M:]


def filter_msgs(msgs, table, fps, ms):
    return [filter_msg(m, table[i // ms], fps[i // ms]) for i, m in enumerate(msgs)]


# ---- the stateless primitive -------------------------------------------------------------------------------------
def _dev(R, ctx, s, fp, out, plain=False):
    import torch

    d = torch.device("cuda", 0)
    n, stride = out["ranges"].shape
    tr = torch.from_numpy(np.ascontiguousarray(out["ranges"])).to(d)
    ti = torch.from_numpy(np.ascontiguousarray(out["intensities"])).to(d)
    tb = torch.from_numpy(out["beam_counts"].view(np.int32)).to(d)
    ta = torch.from_numpy(out["angle_increment"]).to(d)
    a = (tr.data_ptr(), ti.data_ptr(), tb.data_ptr(), ta.data_ptr(), n, stride)
    if plain:
        ctx.scan_filter_batch_dev(s, *a)
    else:
        ctx.scan_filter_footprint_batch_dev(s, fp, *a)
    torch.cuda.synchronize()
    return tr.cpu().numpy(), ti.cpu().numpy()


def _synth_rows(rng, mode_a):
    """rows of beam counts M in {2, 3, 4095, 4096, 8191, 8192}, Mode A (inc = fl(2 pi / M), +inf empty bins) or Mode B
    (inc = fl(2 pi / (M - 1)))"""
    Ms = np.array([2, 3, 4095, 4096, 8191, 8192], np.uint32)
    r = rng.uniform(0.1, 9.0, (len(Ms), 8192)).astype(np.float32)
    if mode_a:
        r[rng.random(r.shape) < 0.1] = np.inf
    inc = (2 * np.pi / (Ms.astype(np.float64) - (0 if mode_a else 1))).astype(np.float32)
    return dict(ranges=r, intensities=rng.uniform(0, 50, r.shape).astype(np.float32), beam_counts=Ms,
                angle_increment=inc)


@pytest.mark.parametrize("mode_a,inv", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_batch_dev_is_the_restatement(R, oracle, mode_a, inv):
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(2 * mode_a + inv)
    removed = 0
    chain = R.scan_filter_settings(**STAGES["chain"])
    for k, fp in enumerate(fleet_footprints(R, 6)):
        for s in (R.scan_filter_settings(), chain):
            for out in (_batch_rows(R, oracle, ctx, mode_a, inv, 10 * k + 2 * mode_a + inv), _synth_rows(rng, mode_a)):
                got_r, got_i = _dev(R, ctx, s, fp, out)
                want = FP.filter_rows(s, fp, out["ranges"], out["intensities"], out["beam_counts"],
                                      out["angle_increment"])
                assert (bits(got_r) == bits(want)).all(), k
                assert (bits(got_i) == bits(out["intensities"])).all()
                removed += int((bits(got_r) != bits(out["ranges"])).sum())
    assert removed > 0
    ctx.close()


@pytest.mark.parametrize("seed", range(4))
def test_batch_dev_random_shapes(R, oracle, seed):
    from test_scan_filters_oracle import _random_settings

    rng = np.random.default_rng(50 + seed)
    ctx = R.Context(0, 8192, 16)
    for t in range(4):
        mode_a = int(rng.integers(0, 2))
        out = _batch_rows(R, oracle, ctx, mode_a, int(rng.integers(0, 2)), 200 + 4 * seed + t) if t % 2 else \
            _synth_rows(rng, mode_a)
        e = _random_settings(rng) if t >= 2 else None
        s = R.scan_filter_settings() if e is None else R.scan_filter_settings(
            mask=list(zip(e.mask_lo, e.mask_hi)), range_lo=e.range_lo, range_hi=e.range_hi,
            intensity_min=e.intensity_min, speckle_window=e.speckle_window,
            speckle_min_neighbours=e.speckle_min_neighbours, speckle_max_diff=e.speckle_max_diff,
            shadow_window=e.shadow_window, shadow_angle=e.shadow_angle)
        fp = random_footprint(R, rng)
        got_r, _ = _dev(R, ctx, s, fp, out)
        want = FP.filter_rows(s, fp, out["ranges"], out["intensities"], out["beam_counts"], out["angle_increment"])
        assert (bits(got_r) == bits(want)).all()
    ctx.close()


def test_null_footprint_is_scan_filter_batch_dev(R, oracle):
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(9)
    for k, kw in enumerate(STAGES.values()):
        s = R.scan_filter_settings(**kw)
        for out in (_batch_rows(R, oracle, ctx, k % 2, k // 2 % 2, 300 + k), _synth_rows(rng, k % 2)):
            a, _ = _dev(R, ctx, s, None, out, plain=True)
            for fp in (None, R.scan_footprint(), R.scan_footprint(pose=(1.0, 2.0, 3.0))):
                b, _ = _dev(R, ctx, s, fp, out)
                assert (bits(a) == bits(b)).all()
    ctx.close()


# ---- sessions ----------------------------------------------------------------------------------------------------
class FootRowPair(RowPair):
    """RowPair with footprints on B (None: B never calls set_scan_footprints)"""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, fps, lidars=None, types=None):
        super().__init__(R, ctx, kind, ans, n, stride, max_nodes, ms, table, lidars=lidars, types=types)
        self.fps = [None] * n if fps is None else list(fps)
        if fps is not None:
            self.B.set_scan_footprints(self.fps)

    def push(self, push, prm, rx=None, dev=False):
        buf, cnt = self.buffers(push)
        fn = self._push_dev if dev else self._push_host
        a = fn(self.A, buf, cnt, prm, rx)
        b = fn(self.B, buf, cnt, flagged(self.R, prm), rx)
        sps = a["scans_per_stream"]
        assert sps.tolist() == b["scans_per_stream"].tolist()
        used = np.flatnonzero(np.arange(self.ms)[None, :] < sps[:, None])
        for k in ("beam_counts", "angle_increment", "scan_begin_ts_us"):
            if k in a:
                assert a[k][used].tobytes() == b[k][used].tobytes(), k
        for i in used:
            M = int(a["beam_counts"][i])
            s = i // self.ms
            want = FP.filter_scan(self.table[s], self.fps[s], a["ranges"][i, :M], a["intensities"][i, :M],
                                  a["angle_increment"][i])
            assert (bits(b["ranges"][i, :M]) == bits(want)).all(), i
            assert (bits(b["intensities"][i, :M]) == bits(a["intensities"][i, :M])).all(), i
            self.changed += int((bits(want) != bits(a["ranges"][i, :M])).sum())

    def compare_after(self, prm):
        R, A, B = self.R, self.A, self.B
        assert filter_msgs(A.laserscan_msgs(prm, 7), self.table, self.fps, self.ms) == \
            B.laserscan_msgs(flagged(R, prm), 7)
        assert A.laserscan_msgs(prm, 7) == B.laserscan_msgs(prm, 7)
        cprm = R.cloud_params(is_new_protocol=prm.is_new_protocol)
        assert A.cloud_msgs(cprm, 7) == B.cloud_msgs(cprm, 7)
        assert A.counters().tobytes() == B.counters().tobytes()


class FootMsgPair(MsgPair):
    """MsgPair with footprints on B"""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, fps, settings=None, types=None):
        super().__init__(R, ctx, kind, ans, n, stride, max_nodes, ms, table, settings=settings, types=types)
        self.fps = list(fps)
        self.B.set_scan_footprints(self.fps)

    def push(self, push, prm, off, rx=None, dev=False, capacity=None, timing=True):
        buf, cnt = self.buffers(push)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        if rx is None:
            out = self.A.push(buf, cnt, prm)
        elif self.kind == "framed":
            out = self.A.push(buf, cnt, prm, rx_us=rx, timing=tm)
        else:
            out = self.A.push(buf, cnt, prm, chunk_bytes=cb, chunk_rx_us=rx, timing=tm)
        exp = filter_msgs(self.A.laserscan_msgs(prm, off), self.table, self.fps, self.ms)
        got = self.push_b(buf, cnt, flagged(self.R, prm), off, rx, tm, cb, dev, capacity)
        assert got["sps"].tolist() == out["scans_per_stream"].tolist()
        self.check(got, exp, capacity)
        return got

    def compare_after(self, prm, cprm, off):
        Pair.compare_after(self, prm, cprm, off)
        exp = filter_msgs(self.A.laserscan_msgs(prm, off), self.table, self.fps, self.ms)
        assert exp == self.B.laserscan_msgs(flagged(self.R, prm), off)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_session_every_answer_type(R, oracle, kind, ans, dev):
    """rows and laserscan_msgs, and push_laserscan_msgs, stamped and unstamped; the device cases with per-stream lidar
    settings mixing Mode A / B and inversion"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 1000)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9400 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    lid = lidar_settings(R, n) if dev else None
    table, fps = fleet_filters(R, n), fleet_footprints(R, n)[::-1]
    rp = FootRowPair(R, ctx, kind, ans, n, stride, 4096, ms, table, fps, lidars=lid)
    mp = FootMsgPair(R, ctx, kind, ans, n, stride, 4096, ms, table, fps, settings=lid)
    if dev:
        prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
        cprm = R.cloud_params(flags=R.CLOUD_PER_STREAM)
    else:
        prm = R.scan_params(int(ans % 2), int(ans > 0x83), int(ans % 3 == 0), 1)
        cprm = R.cloud_params(is_new_protocol=int(ans % 2))
    for t, push in enumerate(pieces):
        rp.push(push, prm, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        rp.compare_after(prm)
        mp.push(push, prm, 11, rx=rx[t] if t % 2 == 0 else None, dev=dev, timing=not dev)
        mp.compare_after(prm, cprm, 11)
    assert rp.changed > 0
    rp.close()
    mp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_several_chunks_and_a_mixed_fleet(R, oracle, dev):
    """23 streams in device chunks of 7 and host chunks of 4: footprints, none, and disabled filter entries with a
    footprint (published as they are)"""
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(oracle, 0x82, n, 1700)]
    rng = np.random.default_rng(29 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = (16 << 20) // 5 + 1
    ctx = R.Context(0, 4096, 7 * ms)
    table = [R.scan_filter_settings() if s % 3 else fleet_filters(R, n)[s] for s in range(n)]
    for s in range(7, 14, 2):
        table[s] = R.scan_filter_settings(enabled=False)
    fps = fleet_footprints(R, n)
    mp = FootMsgPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fps)
    rp = FootRowPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fps)
    prm = R.scan_params(0, 1, 0, 1)
    for push in pieces:
        mp.push(push, prm, 42, dev=dev)
        mp.compare_after(prm, R.cloud_params(), 42)
        rp.push(push, prm, dev=dev)
        rp.compare_after(prm)
    assert rp.changed > 0
    mp.close()
    rp.close()
    ctx.close()


def test_masked_update_applies_from_the_next_push(R, oracle):
    n, ms = 5, 3
    rng = np.random.default_rng(43)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x84, n, 5400, rng)
    ctx = R.Context(0, 4096, n * ms)
    table = [R.scan_filter_settings()] * n
    rp = FootRowPair(R, ctx, "framed", 0x84, n, stride, 4096, ms, table, [R.scan_footprint()] * n)
    prm = R.scan_params(1, 0, 0, 1)
    mask = np.array([1, 0, 1, 0, 1], np.uint8)
    fleet = fleet_footprints(R, n)
    for t, push in enumerate(pieces):
        rp.push(push, prm)
        rp.compare_after(prm)
        new = fleet[t % n: t % n + 1] * n
        rp.B.set_scan_footprints(new, mask=mask if t % 2 else None)
        rp.fps = [new[s] if (not t % 2 or mask[s]) else rp.fps[s] for s in range(n)]
    assert rp.changed > 0
    rp.close()
    ctx.close()


def test_refused_update_leaves_the_table(R, oracle):
    n, ms = 4, 3
    rng = np.random.default_rng(47)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 5500, rng)
    ctx = R.Context(0, 4096, n * ms)
    fps = fleet_footprints(R, n)
    rp = FootRowPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fps)
    prm = R.scan_params(1, 0, 0, 1)
    for t, push in enumerate(pieces):
        kw = BAD[t % len(BAD)]
        with pytest.raises(R.RplError) as e:
            rp.B.set_scan_footprints(fps[:n - 1] + [make(R.scan_footprint, kw)], mask=[1, 0, 1, 1])
        assert e.value.code == R.RESULT_INVALID_DATA
        rp.push(push, prm)
        rp.compare_after(prm)
    assert rp.changed > 0
    rp.close()
    ctx.close()


def test_never_set_is_the_filter_chain(R, oracle):
    """a session that never calls set_scan_footprints filters as the chain without a footprint does"""
    n, ms = 6, 3
    rng = np.random.default_rng(53)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x83, n, 5600, rng)
    ctx = R.Context(0, 4096, n * ms)
    rp = FootRowPair(R, ctx, "framed", 0x83, n, stride, 4096, ms, fleet_filters(R, n), None)
    prm = R.scan_params(1, 1, 1, 1)
    for push in pieces:
        rp.push(push, prm)
        rp.compare_after(prm)
    assert rp.changed > 0
    rp.close()
    ctx.close()


def test_argument_checks(R, oracle):
    import ctypes

    import torch

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    fn = L.rpl_capsule_stream_set_scan_footprints
    arr = (R.ScanFootprint * n)(*[R.scan_footprint()] * n)
    # the first call must set every stream; a null table
    m = np.array([1, 0, 1], np.uint8)
    assert fn(fr._h, ctypes.cast(arr, ctypes.c_void_p), ctypes.c_void_p(m.ctypes.data)) == bad
    assert fn(fr._h, None, None) == bad
    for kw in BAD:
        with pytest.raises(R.RplError) as e:
            fr.set_scan_footprints([R.scan_footprint()] * (n - 1) + [make(R.scan_footprint, kw)])
        assert e.value.code == bad
    for kw in GOOD:
        fr.set_scan_footprints([make(R.scan_footprint, kw)] * n)
    fr.set_scan_footprints([make(R.scan_footprint, BAD[0])] * n, mask=[0, 0, 0])
    # the stateless call's checks
    d = torch.device("cuda", 0)
    rows = torch.zeros((4, 8192), dtype=torch.float32, device=d)
    beams = torch.ones(4, dtype=torch.int32, device=d)
    inc = torch.ones(4, dtype=torch.float32, device=d)
    s = R.scan_filter_settings()
    for kw in BAD:
        with pytest.raises(R.RplError) as e:
            ctx.scan_filter_footprint_batch_dev(s, make(R.scan_footprint, kw), rows.data_ptr(), rows.data_ptr(),
                                                beams.data_ptr(), inc.data_ptr(), 4, 8192)
        assert e.value.code == bad
    torch.cuda.synchronize()
    assert (rows == 0).all()
    fr.close()
    ctx.close()
