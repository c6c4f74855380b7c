"""LaserScans re-gridded from the projected clouds on the device (rpl_rescan_batch_dev, rpl_capsule_stream_set_rescans,
rpl_capsule_stream_rescan_msgs[_dev]) against their definition, oracle/rescan_oracle.py.

The stateless call must be Q of the cloud tests/scan_cloud_transform_oracle.py projects from each row, bit for bit.  A
session's message of slot i must be Q with stream s's entry of the message scan_cloud_msgs gives slot i on the same
session (None where that has none, or the entry is disabled)."""
import math

import numpy as np
import pytest

import scan_cloud_transform_oracle as SCT
from oracle import cdr_oracle as CDR
from oracle import rescan_oracle as RQ
from oracle import scan_cloud_oracle as SC
from test_gpu_scan_cloud import CUTOFFS, GUARD, _with_holes, check_packed
from test_gpu_scan_cloud_transforms import XfPair, capi_entry, fleet_transforms, frames_for
from test_gpu_scan_filters import fleet_filters, flagged
from test_gpu_scan_footprints import _synth_rows, fleet_footprints
from test_gpu_stream_push_msgs import lidar_settings, pieces_for, receive_times

pytestmark = pytest.mark.gpu

XF = SCT.PER_STREAM_TRANSFORMS
TWO_PI = 2 * math.pi
# (angle_min, angle_max, angle_increment): 1, 7, 360, 4096 and 8192 bins over the full circle or part of it
GRIDS = [(-math.pi, math.pi, 7.0), (-1.0, 1.0, 0.29), (-math.pi, math.pi, math.pi / 180), (-math.pi, math.pi,
         TWO_PI / 4095.5), (-math.pi, math.pi, TWO_PI / 8191.5), (-0.5, 1.2, 0.01), (0.3, 2.9, 0.0005)]
TRANSFORMS = {
    "none": None,
    "identity": SCT.transform(),
    "offset": SCT.transform((0.3, -0.2, 0.5)),
    "tilted": SCT.transform((0.1, 0.0, 0.4), (math.sin(0.15), 0.0, 0.0, math.cos(0.15))),
    "upside_down": SCT.transform((0.0, 0.0, 0.2), (1.0, 0.0, 0.0, 0.0)),
}


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def capi_settings(R, s):
    return R.rescan_settings(s.angle_min, s.angle_max, s.angle_increment, s.range_min, s.range_max, s.min_height,
                             s.max_height, s.use_inf, s.inf_epsilon, s.scan_time, s.enabled)


def test_grid_sizes():
    assert [RQ.ranges_size(RQ.settings(*g)) for g in GRIDS[:5]] == [1, 7, 360, 4096, 8192]


def _cloud_xyz(rec):
    w = rec.view("<u4").reshape(rec.shape[0], rec.shape[1] // 4)
    return w[:, 0].view(np.float32), w[:, 1].view(np.float32), w[:, 2].view(np.float32)


def _batch(R, ctx, s, p, e, out, lo, hi):
    import torch

    d = torch.device("cuda", 0)
    n, stride = out["ranges"].shape
    bins = RQ.ranges_size(s)
    t = {k: torch.from_numpy(np.ascontiguousarray(out[k])).to(d) for k in ("ranges", "angle_increment")}
    tb = torch.from_numpy(np.ascontiguousarray(out["beam_counts"]).view(np.int32)).to(d)
    o = torch.full((n * bins + 16,), -7.0, dtype=torch.float32, device=d)
    torch.cuda.synchronize()
    ctx.rescan_batch_dev(capi_settings(R, s), R.scan_cloud_params(p.channels, p.range_cutoff),
                         None if e is None else capi_entry(R, e), t["ranges"].data_ptr(), None, tb.data_ptr(),
                         t["angle_increment"].data_ptr(), lo, hi, n, stride, o.data_ptr())
    torch.cuda.synchronize()
    got = o.cpu().numpy()
    assert (got[n * bins:] == np.float32(-7.0)).all()
    return got[: n * bins].reshape(n, bins)


def _want_rows(s, p, e, out, lo, hi):
    rows = []
    for k in range(out["ranges"].shape[0]):
        M = int(out["beam_counts"][k])
        rec = SCT.project(p, out["ranges"][k, :M], out["intensities"][k, :M], out["angle_increment"][k], 0.0, lo, hi,
                          e)
        rows.append(RQ.regrid(s, *_cloud_xyz(rec)))
    return np.stack(rows)


@pytest.mark.parametrize("xf", list(TRANSFORMS))
def test_batch_dev_is_the_restatement(R, xf):
    """every grid, use_inf on and off, height bands that cut the tilted cloud, rows with NaN and +-inf"""
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(sorted(TRANSFORMS).index(xf) + 40)
    e = TRANSFORMS[xf]
    hit = 0
    for k, g in enumerate(GRIDS):
        out = _with_holes(rng, _synth_rows(rng, k % 2))
        band = (0.3, 0.6) if k % 3 == 1 else (-0.05, 1e-3) if k % 3 == 2 else (-RQ.FLT_MAX, RQ.FLT_MAX)
        s = RQ.settings(*g, range_min=float(k % 2) * 0.5, range_max=8.0 + k, min_height=band[0], max_height=band[1],
                        use_inf=k % 2 == 0, inf_epsilon=0.25 * k)
        p = SC.params(SCT.VIEWPOINT | 0x03 if e is not None else 0x03, CUTOFFS[k % len(CUTOFFS)])
        got = _batch(R, ctx, s, p, e, out, 0.15, 12.0)
        want = _want_rows(s, p, e, out, 0.15, 12.0)
        assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist(), (xf, g)
        hit += int((got != RQ.seed(s)).sum())
    assert hit > 0
    ctx.close()


def test_batch_dev_refusals(R):
    import ctypes

    import torch

    ctx = R.Context(0, 4096, 4)
    d = torch.device("cuda", 0)
    rows = torch.zeros((4, 4096), dtype=torch.float32, device=d)
    cnt = torch.ones(4, dtype=torch.int32, device=d)
    o = torch.full((4 * 8192 + 8,), -7.0, dtype=torch.float32, device=d)
    torch.cuda.synchronize()
    L = R.lib()
    bad = [dict(angle_increment=0.0), dict(angle_min=1.0, angle_max=1.0), dict(angle_max=math.inf),
           dict(range_min=-0.1), dict(range_min=5.0, range_max=4.0), dict(min_height=1.0, max_height=0.5),
           dict(inf_epsilon=-1.0), dict(scan_time=math.nan), dict(angle_increment=TWO_PI / 8192.5)]
    cp = R.scan_cloud_params()
    for b in bad:
        s = R.rescan_settings(**b)
        assert L.rpl_rescan_batch_dev(ctx._h, ctypes.byref(s), ctypes.byref(cp), None, rows.data_ptr(), None,
                                      cnt.data_ptr(), rows.data_ptr(), 0.15, 40.0, 4, 4096, o.data_ptr(),
                                      None) == R.RESULT_INVALID_DATA, b
    ok = R.rescan_settings()
    for c, t in ((R.scan_cloud_params(0x10), None), (R.scan_cloud_params(XF), None),
                 (R.scan_cloud_params(0x03, math.nan), None),
                 (R.scan_cloud_params(0x03), R.scan_cloud_transform((2000.0, 0, 0)))):
        assert L.rpl_rescan_batch_dev(ctx._h, ctypes.byref(ok), ctypes.byref(c), None if t is None else ctypes.byref(t),
                                      rows.data_ptr(), None, cnt.data_ptr(), rows.data_ptr(), 0.15, 40.0, 4, 4096,
                                      o.data_ptr(), None) == R.RESULT_INVALID_DATA
    torch.cuda.synchronize()
    assert (o.cpu().numpy() == np.float32(-7.0)).all()
    ctx.close()


# ---- sessions ----------------------------------------------------------------------------------------------------
def fleet_rescans(rng, n):
    """entries over every grid, with every fourth disabled"""
    out = []
    for s in range(n):
        g = GRIDS[(s + int(rng.integers(0, len(GRIDS)))) % len(GRIDS)]
        lo = float(rng.uniform(-0.3, 0.0))
        out.append(RQ.settings(*g, range_min=float(rng.uniform(0, 0.5)), range_max=float(rng.uniform(4, 12)),
                               min_height=lo, max_height=float(rng.uniform(0.0, 0.6)), use_inf=s % 2 == 0,
                               inf_epsilon=float(rng.uniform(0, 1)), scan_time=float(rng.uniform(0.05, 0.2)),
                               enabled=s % 4 != 3))
    return out


def rescan_dev(R, X, prm, cp, off, capacity=None):
    import torch

    ns = X.n_streams * X.max_scans
    cap = ns * ((288 + 36 + 4 * 8192 + 15) // 16 * 16) if capacity is None else capacity
    d = torch.device("cuda", 0)
    store = torch.full((cap + 256,), GUARD, dtype=torch.uint8, device=d)
    offs = torch.full((ns,), -1, dtype=torch.int64, device=d)
    sizes = torch.full((ns,), -1, dtype=torch.int32, device=d)
    total = torch.full((1,), -1, dtype=torch.int64, device=d)
    torch.cuda.synchronize()
    X.rescan_msgs_dev(prm, cp, off, store.data_ptr(), cap, offs.data_ptr(), sizes.data_ptr(), total.data_ptr())
    torch.cuda.synchronize()
    return dict(msgs=store.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]))


def rescanned(clouds, entries, ms):
    return [None if c is None else RQ.Q(entries[i // ms], CDR.parse_pointcloud2(c)) for i, c in enumerate(clouds)]


class RescanPair(XfPair):
    def set_rescans(self, entries, mask=None):
        if mask is None:
            self.rescans = list(entries)
        else:
            for s in np.flatnonzero(mask):
                self.rescans[s] = entries[s]
        for x in (self.A, self.B):
            x.set_rescans([capi_settings(self.R, e) for e in entries], mask)

    def compare_rescans(self, prm, off, cps, dev=False):
        """each session's rescan_msgs against Q of its own scan_cloud_msgs, slot by slot"""
        R = self.R
        for k, q in enumerate((prm, flagged(R, prm))):
            X = self.A if k else self.B
            for cp in cps:
                want = rescanned(X.scan_cloud_msgs(q, cp, off), self.rescans, self.ms)
                if dev:
                    check_packed(rescan_dev(R, X, q, cp, off), want, 1 << 62)
                else:
                    assert X.rescan_msgs(q, cp, off) == want
                self.msgs += sum(w is not None for w in want)


def _cps(R):
    return [R.scan_cloud_params(0x03), R.scan_cloud_params(XF | 0x1F, 6.0), R.scan_cloud_params(XF | 0x0C, 0.0)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", [("framed", 0x85), ("bytes", 0x82), ("bytes", 0x81)])
def test_session_messages(R, oracle, kind, ans, dev):
    """per-stream filters and footprints, transform and rescan entries with disabled ones, masked updates between
    pushes, stamped and unstamped pushes; the device cases with per-stream lidars"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 8100)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9700 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    lid = lidar_settings(R, n) if dev else None
    cp = RescanPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n), lidars=lid)
    cp.msgs = 0
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n))
    cp.set_rescans(fleet_rescans(rng, n))
    prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                int(ans % 3 == 0), 1)
    for t, push in enumerate(pieces):
        cp.push(push, prm, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        cp.compare_rescans(prm, 987_654_321 if t % 2 else -5, _cps(R), dev=dev)
        cp.set_rescans(fleet_rescans(rng, n), (rng.random(n) < 0.5).astype(np.uint8))
        cp.set_transforms(fleet_transforms(rng, n), frames_for(n, t + 1), (rng.random(n) < 0.5).astype(np.uint8))
    assert cp.msgs > 0
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session(R, oracle, dev):
    from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
    from test_gpu_stream_stamps import _streams

    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    n, ms = len(types), 3
    rng = np.random.default_rng(61 + dev)
    st = [_streams(oracle, t, 1, 900 + s)[0].reshape(-1) for s, t in enumerate(types)]
    pieces, _ = _pieces_from_cuts(st, [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in st])
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 4096, n * ms)
    cp = RescanPair(R, ctx, "bytes", 0, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n), types=types)
    cp.msgs = 0
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n))
    cp.set_rescans(fleet_rescans(rng, n))
    prm = R.scan_params(1, 0, 1, 1)
    for push in pieces:
        cp.push(push, prm, dev=dev)
        cp.compare_rescans(prm, 5, _cps(R), dev=dev)
    assert cp.msgs > 0
    cp.close()
    ctx.close()


def test_emptied_scans_give_seeded_messages(R, oracle):
    """a range window that removes every beam: every enabled stream's slots still have messages, every beam its seed"""
    n, ms = 4, 3
    rng = np.random.default_rng(77)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9800, rng)
    ctx = R.Context(0, 4096, n * ms)
    empty = [R.scan_filter_settings(range_lo=100.0, range_hi=200.0)] * n
    cp = RescanPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, empty, fleet_footprints(R, n))
    cp.msgs = 0
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n))
    cp.set_rescans([RQ.settings(use_inf=s % 2 == 0, range_max=5.0, enabled=s != 2) for s in range(n)])
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    seen = 0
    for push in pieces:
        cp.push(push, prm)
        got = cp.B.rescan_msgs(prm, R.scan_cloud_params(XF | 0x03), 0)
        clouds = cp.B.scan_cloud_msgs(prm, R.scan_cloud_params(XF | 0x03), 0)
        for i, (g, c) in enumerate(zip(got, clouds)):
            if c is None or i // ms == 2:
                assert g is None
                continue
            assert CDR.parse_pointcloud2(c)["width"] == 0
            m = CDR.parse_laserscan(g)
            assert m["ranges"].shape == (360,) and (m["ranges"] == RQ.seed(cp.rescans[i // ms])).all()
            seen += 1
    assert seen > 0
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """exactly met and one byte short: all or nothing"""
    n, ms = 5, 3
    rng = np.random.default_rng(271 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9900, rng)
    ctx = R.Context(0, 4096, n * ms)
    cp = RescanPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n, 4))
    cp.set_rescans(fleet_rescans(rng, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    q = R.scan_cloud_params(XF | 0x03)
    tested = 0
    for push in pieces:
        cp.push(push, prm)
        want = rescanned(cp.B.scan_cloud_msgs(prm, q, 3), cp.rescans, ms)
        full = check_packed(rescan_dev(R, cp.B, prm, q, 3), want, 1 << 62)
        if full == 0:
            continue
        for cap in (full, full - 1):
            if dev:
                check_packed(rescan_dev(R, cp.B, prm, q, 3, capacity=cap), want, cap)
            else:
                store = np.full(cap + 256, GUARD, np.uint8)
                res = cp.B.rescan_msgs(prm, q, 3, msgs=store[:cap], packed=True)
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


def test_session_refusals_and_a_refused_set_changes_nothing(R, oracle):
    import ctypes

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    bad = R.RESULT_INVALID_DATA
    prm = R.scan_params(1, 0, 0, 1)
    fr.push(np.zeros((n, 8, 84), np.uint8), np.zeros(n, np.uint32), prm)
    with pytest.raises(R.RplError) as e:  # before the first set call
        fr.rescan_msgs(prm, R.scan_cloud_params())
    assert e.value.code == bad
    L = R.lib()
    ok = [R.rescan_settings(), R.rescan_settings(enabled=False), R.rescan_settings(-1.0, 1.0, 0.01)]
    arr = (R.capi.RescanSettings * n)(*ok)
    half = np.array([1, 0, 1], np.uint8)
    assert L.rpl_capsule_stream_set_rescans(fr._h, ctypes.cast(arr, ctypes.c_void_p), half.ctypes.data) == bad
    assert L.rpl_capsule_stream_set_rescans(fr._h, None, None) == bad
    fr.set_rescans(ok)
    before = fr.rescan_msgs(prm, R.scan_cloud_params())
    for b in (dict(angle_increment=0.0), dict(range_min=-1.0), dict(min_height=2.0, max_height=1.0),
              dict(inf_epsilon=math.nan), dict(angle_increment=1e-5)):
        t = list(ok)
        t[2] = R.rescan_settings(**b)
        with pytest.raises(R.RplError) as ex:
            fr.set_rescans(t)
        assert ex.value.code == bad
    # a disabled entry is not read
    fr.set_rescans([ok[0], R.rescan_settings(angle_increment=0.0, enabled=False), ok[2]])
    assert fr.rescan_msgs(prm, R.scan_cloud_params()) == before
    for c in (R.scan_cloud_params(0x10), R.scan_cloud_params(XF), R.scan_cloud_params(0x13, math.nan)):
        with pytest.raises(R.RplError):
            fr.rescan_msgs(prm, c)
    fr.close()
    ctx.close()
