"""Projected clouds in a target frame on the device (rpl_scan_cloud_transform_batch_dev,
rpl_capsule_stream_set_scan_cloud_transforms, RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS on scan_cloud_msgs[_dev] and
push_scan_cloud_msgs[_dev]) against their definition, tests/scan_cloud_transform_oracle.py.

The stateless call must be the restatement bit for bit.  A session's message of slot i must be P with stream s's entry
and target frame of the laserscan_msgs message of the same slot on a twin session; a push that returns both sets must
agree with a twin that pushes and then replays, as without a transform."""
import math

import numpy as np
import pytest

import scan_cloud_transform_oracle as SCT
from oracle import cdr_oracle as CDR
from oracle import scan_cloud_oracle as SC
from test_gpu_scan_cloud import CUTOFFS, GUARD, CloudPair, _with_holes, check_packed
from test_gpu_scan_filters import _batch_rows, fleet_filters, flagged
from test_gpu_scan_footprints import _synth_rows, fleet_footprints
from test_gpu_stream_push_msgs import lidar_settings, pieces_for, receive_times
from test_gpu_stream_push_scan_cloud_msgs import ScanCloudPair, fleet

pytestmark = pytest.mark.gpu

XF = SCT.PER_STREAM_TRANSFORMS


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _quat(rng):
    q = rng.normal(size=4)
    return tuple(float(v) for v in q / np.linalg.norm(q) * math.sqrt(1 + rng.uniform(-9e-4, 9e-4)))


def random_entry(rng, enabled=True):
    return SCT.transform(rng.uniform(-20, 20, 3), _quat(rng), enabled)


def capi_entry(R, e):
    return R.scan_cloud_transform(e.translation, e.rotation, e.enabled)


def frames_for(n, k=0):
    """target frames of 0..255 characters"""
    lens = [0, 1, 9, 64, 254, 255, 3, 17]
    return ["f%d_" % s + "x" * max(0, lens[(s + k) % len(lens)] - len("f%d_" % s)) if lens[(s + k) % len(lens)] else ""
            for s in range(n)]


def fleet_transforms(rng, n):
    """enabled entries with every third disabled"""
    return [random_entry(rng, s % 3 != 1) for s in range(n)]


# ---- the stateless primitive -------------------------------------------------------------------------------------
def _xf_batch_dev(R, ctx, p, out, ti, lo, hi, e, plain=False):
    import torch

    d = torch.device("cuda", 0)
    n, stride = out["ranges"].shape
    step = SCT.point_step(p.channels)
    t = {k: torch.from_numpy(np.ascontiguousarray(out[k])).to(d) for k in ("ranges", "intensities", "angle_increment")}
    tb = torch.from_numpy(np.ascontiguousarray(out["beam_counts"]).view(np.int32)).to(d)
    tt = None if ti is None else torch.from_numpy(ti).to(d)
    pts = torch.full((n * stride * step + 64,), GUARD, dtype=torch.uint8, device=d)
    cnt = torch.full((n,), -1, dtype=torch.int32, device=d)
    torch.cuda.synchronize()
    args = (t["ranges"].data_ptr(), t["intensities"].data_ptr(), tb.data_ptr(), t["angle_increment"].data_ptr(),
            None if tt is None else tt.data_ptr(), lo, hi, n, stride, pts.data_ptr(), cnt.data_ptr())
    cp = R.scan_cloud_params(p.channels, p.range_cutoff)
    if plain:
        ctx.scan_cloud_batch_dev(cp, *args)
    else:
        ctx.scan_cloud_transform_batch_dev(cp, None if e is None else capi_entry(R, e), *args)
    torch.cuda.synchronize()
    return pts.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _check_xf_rows(R, ctx, p, out, ti, lo, hi, e):
    n, stride = out["ranges"].shape
    step = SCT.point_step(p.channels)
    pts, cnt = _xf_batch_dev(R, ctx, p, out, ti, lo, hi, e)
    want, wcnt = SCT.project_rows(p, out["ranges"], out["intensities"], out["beam_counts"], out["angle_increment"],
                                  ti, lo, hi, e)
    assert cnt.tolist() == wcnt.tolist()
    for s in range(n):
        row = pts[s * stride * step: s * stride * step + int(cnt[s]) * step]
        assert row.tobytes() == want[s].tobytes(), s
    assert (pts[n * stride * step:] == GUARD).all()
    return int(wcnt.sum())


@pytest.mark.parametrize("mode_a,inv", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_batch_dev_every_channel_set(R, oracle, mode_a, inv):
    """random transforms (every fourth disabled) over all 32 channel sets, the cutoffs, rows with NaN and +inf, M in
    [1, 8192]"""
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(500 + 2 * mode_a + inv)
    kept = 0
    for ch in range(32):
        base = _batch_rows(R, oracle, ctx, mode_a, inv, 3 * ch + mode_a) if ch % 2 else _synth_rows(rng, mode_a)
        out = _with_holes(rng, base)
        n = out["ranges"].shape[0]
        ti = None if ch % 3 == 0 else rng.uniform(1e-6, 1e-3, n).astype(np.float32)
        e = random_entry(rng, ch % 4 != 3)
        kept += _check_xf_rows(R, ctx, SC.params(ch, CUTOFFS[ch % len(CUTOFFS)]), out, ti, 0.15, 12.0, e)
    assert kept > 0
    ctx.close()


def test_batch_dev_null_and_identity(R, oracle):
    """a NULL transform is rpl_scan_cloud_batch_dev byte for byte; identity gives its records too (ranges > 0)"""
    ctx = R.Context(0, 8192, 16)
    rng = np.random.default_rng(61)
    for ch in range(16):
        out = _with_holes(rng, _synth_rows(rng, ch % 2))
        ti = rng.uniform(1e-6, 1e-3, out["ranges"].shape[0]).astype(np.float32)
        p = SC.params(ch, CUTOFFS[ch % len(CUTOFFS)])
        plain = _xf_batch_dev(R, ctx, p, out, ti, 0.15, 12.0, None, plain=True)
        null = _xf_batch_dev(R, ctx, p, out, ti, 0.15, 12.0, None)
        ident = _xf_batch_dev(R, ctx, p, out, ti, 0.15, 12.0, SCT.transform())
        for got in (null, ident):
            assert got[0].tobytes() == plain[0].tobytes() and got[1].tolist() == plain[1].tolist()
    ctx.close()


def test_batch_dev_refusals(R, oracle):
    import torch

    ctx = R.Context(0, 4096, 4)
    d = torch.device("cuda", 0)
    rows = torch.zeros((4, 4096), dtype=torch.float32, device=d)
    cnt = torch.ones(4, dtype=torch.int32, device=d)
    pts = torch.full((4 * 4096 * 40 + 8,), GUARD, dtype=torch.uint8, device=d)
    a = (rows.data_ptr(), rows.data_ptr(), cnt.data_ptr(), rows.data_ptr(), None, 0.15, 40.0, 4, 4096,
         pts.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    bad = R.RESULT_INVALID_DATA
    L = R.lib()
    cases = [(R.scan_cloud_params(0x10), None), (R.scan_cloud_params(XF), R.scan_cloud_transform()),
             (R.scan_cloud_params(XF | 0x13), None), (R.scan_cloud_params(0x20), R.scan_cloud_transform()),
             (R.scan_cloud_params(0x13, math.nan), R.scan_cloud_transform())]
    for e, frame, good in _limits():
        if frame is not None and frame != "":
            continue
        if not good:
            cases.append((R.scan_cloud_params(0x13), capi_entry(R, e)))
    import ctypes

    for p, t in cases:
        rc = L.rpl_scan_cloud_transform_batch_dev(ctx._h, ctypes.byref(p), None if t is None else ctypes.byref(t), *a,
                                                  None)
        assert rc == bad, (p.channels, None if t is None else list(t.translation) + list(t.rotation))
    # the viewpoint with a transform, a disabled one included, is accepted
    for t in (R.scan_cloud_transform(), R.scan_cloud_transform((math.nan,) * 3, enabled=False)):
        assert L.rpl_scan_cloud_transform_batch_dev(ctx._h, ctypes.byref(R.scan_cloud_params(0x1F)),
                                                    ctypes.byref(t), *a, None) == R.RESULT_OK
    torch.cuda.synchronize()
    assert (pts.cpu().numpy()[4 * 4096 * 40:] == GUARD).all()
    ctx.close()


def _limits():
    """(entry, frame, ok) on both sides of every bound; frame None: the stateless call's"""
    T = SCT.transform
    out = [(T(), "a" * 255, True), (T(), "a" * 256, False), (T(), "", True),
           (T(rotation=(0, 0, 0, math.sqrt(1.000999))), "", True), (T(rotation=(0, 0, 0, math.sqrt(1.001001))), "", False),
           (T(rotation=(0, 0, 0, math.sqrt(0.999001))), "", True), (T(rotation=(0, 0, 0, math.sqrt(0.998999))), "", False),
           (T((1000.0, -1000.0, 1000.0)), "", True), (T((1000.001, 0, 0)), "", False), (T((0, 0, -1000.001)), "", False),
           (T((math.nan, 0, 0)), "", False), (T((0, math.inf, 0)), "", False), (T(rotation=(0, 0, math.nan, 1)), "", False)]
    for e, f, good in out:
        assert SCT.transform_ok(e, f) == good
    return out


# ---- sessions ----------------------------------------------------------------------------------------------------
PARAMS = [SC.params(SC.DEFAULT), SC.params(SC.CHANNELS | SCT.VIEWPOINT, 6.0), SC.params(SCT.VIEWPOINT),
          SC.params(SC.TIMESTAMP | SC.DISTANCE, 0.0)]


def xf_params(R, p):
    return R.scan_cloud_params(p.channels | XF, p.range_cutoff)


def projected_xf(msgs, p, entries, frames, ms):
    return [None if m is None else SCT.P(p, CDR.parse_laserscan(m), entries[i // ms], frames[i // ms])
            for i, m in enumerate(msgs)]


def xf_dev(R, X, prm, cp, off, capacity=None):
    import torch

    ns = X.n_streams * X.max_scans
    cap = ns * ((R.capi._scan_cloud_bound(cp.channels, X.max_nodes) + 15) // 16 * 16) if capacity is None else capacity
    d = torch.device("cuda", 0)
    store = torch.full((cap + 256,), GUARD, dtype=torch.uint8, device=d)
    offs = torch.full((ns,), -1, dtype=torch.int64, device=d)
    sizes = torch.full((ns,), -1, dtype=torch.int32, device=d)
    total = torch.full((1,), -1, dtype=torch.int64, device=d)
    torch.cuda.synchronize()
    X.scan_cloud_msgs_dev(prm, cp, off, store.data_ptr(), cap, offs.data_ptr(), sizes.data_ptr(), total.data_ptr())
    torch.cuda.synchronize()
    return dict(msgs=store.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]))


class XfPair(CloudPair):
    """CloudPair whose sessions both carry the transform table"""

    def set_transforms(self, entries, frames, mask=None):
        if mask is None:
            self.entries, self.frames = list(entries), list(frames)
        else:
            for s in np.flatnonzero(mask):
                self.entries[s], self.frames[s] = entries[s], frames[s]
        for x in (self.A, self.B):
            x.set_scan_cloud_transforms([capi_entry(self.R, e) for e in entries],
                                        [f if e.enabled else None for e, f in zip(entries, frames)], mask)

    def compare_xf(self, prm, off, dev=False, params=PARAMS):
        R = self.R
        for k, q in enumerate((prm, flagged(R, prm))):
            X, Y = (self.A, self.B) if k else (self.B, self.A)
            scans = Y.laserscan_msgs(q, off)
            for p in params:
                want = projected_xf(scans, p, self.entries, self.frames, self.ms)
                if dev:
                    check_packed(xf_dev(R, X, q, xf_params(R, p), off), want, 1 << 62)
                else:
                    assert X.scan_cloud_msgs(q, xf_params(R, p), off) == want
                for w in want:
                    if w is not None:
                        self.points += CDR.parse_pointcloud2(w)["width"]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", [("framed", 0x85), ("bytes", 0x82), ("bytes", 0x81), ("framed", 0x84)])
def test_session_messages(R, oracle, kind, ans, dev):
    """mixed enabled and disabled entries, target frames of 0..255 characters, masked updates and a set_frames between
    pushes, filters with footprints; the device cases with per-stream lidars mixing Mode A / B and inversion"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 7000)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9700 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    lid = lidar_settings(R, n) if dev else None
    cp = XfPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n), lidars=lid)
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n))
    prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                int(ans % 3 == 0), 1)
    for t, push in enumerate(pieces):
        cp.push(push, prm, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        cp.compare_xf(prm, 987_654_321 if t % 2 else -5, dev=dev)
        mask = (rng.random(n) < 0.5).astype(np.uint8)
        cp.set_transforms(fleet_transforms(rng, n), frames_for(n, t + 1), mask)
        if t == 1:
            for x in (cp.A, cp.B):
                x.set_frames(["scan_%d" % s for s in range(n)])
    assert cp.points > 0
    cp.close()
    ctx.close()


def test_identity_to_the_laserscan_frame_is_the_call_without_the_bit(R, oracle):
    n, ms = 5, 3
    rng = np.random.default_rng(91)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9650, rng)
    ctx = R.Context(0, 4096, n * ms)
    cp = XfPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    names = ["laser_%d" % s for s in range(n)]
    for x in (cp.A, cp.B):
        x.set_frames(names)
    cp.set_transforms([SCT.transform(enabled=s % 2 == 0) for s in range(n)], names)
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    for push in pieces:
        cp.push(push, prm)
        for ch in range(16):
            p = R.scan_cloud_params(ch, CUTOFFS[ch % len(CUTOFFS)])
            assert cp.B.scan_cloud_msgs(prm, xf_params(R, p), 3) == cp.B.scan_cloud_msgs(prm, p, 3)
            a, b = xf_dev(R, cp.B, prm, xf_params(R, p), 3), xf_dev(R, cp.B, prm, p, 3)
            for k in ("msg_offsets", "msg_sizes"):
                assert a[k].tolist() == b[k].tolist()
            assert a["total_bytes"] == b["total_bytes"] and a["msgs"][:a["total_bytes"]].tobytes() == \
                b["msgs"][:b["total_bytes"]].tobytes()
    cp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """exactly met and one byte short, with long target frames and the viewpoint: all or nothing"""
    n, ms = 5, 3
    rng = np.random.default_rng(171 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9900, rng)
    ctx = R.Context(0, 4096, n * ms)
    cp = XfPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n, 4))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    p = SC.params(SC.CHANNELS | SCT.VIEWPOINT)
    q = xf_params(R, p)
    tested = 0
    for push in pieces:
        cp.push(push, prm)
        want = projected_xf(cp.A.laserscan_msgs(prm, 3), p, cp.entries, cp.frames, ms)
        full = check_packed(xf_dev(R, cp.B, prm, q, 3), want, 1 << 62)
        if full == 0:
            continue
        for cap in (full, full - 1):
            if dev:
                check_packed(xf_dev(R, cp.B, prm, q, 3, capacity=cap), want, cap)
            else:
                store = np.full(cap + 256, GUARD, np.uint8)
                res = cp.B.scan_cloud_msgs(prm, q, 3, msgs=store[:cap], packed=True)
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


# ---- the push that returns both sets ------------------------------------------------------------------------------
class XfScanCloudPair(ScanCloudPair):
    """ScanCloudPair with the transform table on both sessions, its cloud buffers sized for the viewpoint"""

    def cloud_big(self, cp):
        return self.n * self.ms * ((self.R.capi._scan_cloud_bound(cp.channels, self.max_nodes) + 15) // 16 * 16)

    def set_transforms(self, entries, frames, mask=None):
        for x in (self.A, self.B):
            x.set_scan_cloud_transforms([capi_entry(self.R, e) for e in entries],
                                        [f if e.enabled else None for e, f in zip(entries, frames)], mask)


def xf_channel_sets(R):
    return [R.scan_cloud_params(XF | 0x03), R.scan_cloud_params(XF | 0x1F, 6.0), R.scan_cloud_params(XF | 0x10),
            R.scan_cloud_params(XF | 0x0C, 0.0)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_push_with_transforms(R, oracle, dev):
    """per-stream lidars with inversion, filters with footprints, masked updates between pushes"""
    n, ms = 7, 3
    rng = np.random.default_rng(300 + dev)
    streams, pieces, stride = pieces_for(oracle, "bytes", 0x85, n, 9960, rng)
    rx = receive_times("bytes", rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = XfScanCloudPair(R, ctx, "bytes", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                        settings=lidar_settings(R, n))
    p.set_transforms(fleet_transforms(rng, n), frames_for(n))
    base = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
    cps = xf_channel_sets(R)
    for t, push in enumerate(pieces):
        prm = flagged(R, base) if t % 2 == 0 else base
        p.push(push, prm, cps[t % 4], 55, rx=rx[t] if t % 2 == 0 else None, dev=dev, timing=False)
        p.compare_after(prm, cps[(t + 1) % 4], 55)
        p.set_transforms(fleet_transforms(rng, n), frames_for(n, t + 3), (rng.random(n) < 0.5).astype(np.uint8))
    assert p.n_msgs > n and p.points > 0
    p.close()
    ctx.close()


def test_push_fleet_in_uneven_chunks_with_long_frames_and_the_viewpoint(R, oracle):
    """23 streams (device chunks of 3, host chunks of 4), frames up to 255 characters, host and device calls
    alternating: the clouds' directory carries and the host form's bound use the target headers"""
    n, ms, pieces, stride, rx, table = fleet(R, oracle, 1500)
    ctx = R.Context(0, 4096, 3 * ms)
    p = XfScanCloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fleet_footprints(R, n))
    rng = np.random.default_rng(1500)
    p.set_transforms(fleet_transforms(rng, n), ["t" * (255 - s) for s in range(n)])
    prm = flagged(R, R.scan_params(0, 1, 0, 1))
    cp = R.scan_cloud_params(XF | 0x1F)
    for t, push in enumerate(pieces):
        p.push(push, prm, cp, 42, rx=rx[t] if t % 2 == 0 else None, dev=(t // 2) % 2 == 1)
        p.compare_after(prm, cp, 42)
    assert p.n_msgs > n and p.empty > 0
    p.close()
    ctx.close()


# ---- refusals -----------------------------------------------------------------------------------------------------
def test_session_refusals_and_a_refused_set_changes_nothing(R, oracle):
    import ctypes

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    bad = R.RESULT_INVALID_DATA
    L = R.lib()
    prm = R.scan_params(1, 0, 0, 1)
    fr.push(np.zeros((n, 8, 84), np.uint8), np.zeros(n, np.uint32), prm)
    # the bit before the first set call; the viewpoint without the bit
    for c in (R.scan_cloud_params(XF), R.scan_cloud_params(0x10), R.scan_cloud_params(0x13)):
        with pytest.raises(R.RplError) as e:
            fr.scan_cloud_msgs(prm, c)
        assert e.value.code == bad
    ok = [R.scan_cloud_transform((1, 2, 3)), R.scan_cloud_transform(enabled=False), R.scan_cloud_transform()]
    frames = ["base_link", None, ""]
    arr = (R.capi.ScanCloudTransform * n)(*ok)
    names = (ctypes.c_char_p * n)(*(None if f is None else f.encode() for f in frames))
    half = np.array([1, 0, 1], np.uint8)
    h = fr._h
    f = L.rpl_capsule_stream_set_scan_cloud_transforms
    # a first call must set every stream; null arguments
    assert f(h, ctypes.cast(arr, ctypes.c_void_p), ctypes.cast(names, ctypes.c_void_p), half.ctypes.data) == bad
    assert f(h, None, ctypes.cast(names, ctypes.c_void_p), None) == bad
    assert f(h, ctypes.cast(arr, ctypes.c_void_p), None, None) == bad
    with pytest.raises(R.RplError):
        fr.scan_cloud_msgs(prm, R.scan_cloud_params(XF))
    fr.set_scan_cloud_transforms(ok, frames)
    before = fr.scan_cloud_msgs(prm, R.scan_cloud_params(XF | 0x1F))
    # every limit refused, the table unchanged: masked bad entries, a null frame of an enabled entry
    for e, frame, good in _limits():
        if good:
            continue
        t = list(ok)
        t[0] = capi_entry(R, e)
        with pytest.raises(R.RplError) as ex:
            fr.set_scan_cloud_transforms(t, [frame, None, ""])
        assert ex.value.code == bad
    with pytest.raises(R.RplError):
        fr.set_scan_cloud_transforms([R.scan_cloud_transform()] * n, [None] * n)
    assert fr.scan_cloud_msgs(prm, R.scan_cloud_params(XF | 0x1F)) == before
    # the bit and the viewpoint are refused everywhere else: the stateless call without a transform, the node calls
    for c in (R.scan_cloud_params(0x10), R.scan_cloud_params(XF | 0x20), R.scan_cloud_params(XF | 0x13, math.nan)):
        with pytest.raises(R.RplError):
            fr.scan_cloud_msgs(prm, c)
    fr.close()
    ctx.close()


def test_calls_without_the_bit_launch_what_they_launched(R, oracle):
    """the same kernels, counted by rpl_ctx_launch_count, before and after the table is set, and with the bit"""
    n, ms = 5, 3
    rng = np.random.default_rng(44)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9600, rng)
    ctx = R.Context(0, 4096, n * ms)
    cp = XfPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(1, 0, 0, 1))
    cp.push(pieces[0], prm)
    p = R.scan_cloud_params(0x0F)

    def launches(c, dev):
        k = ctx.launch_count
        if dev:
            xf_dev(R, cp.B, prm, c, 0)
        else:
            cp.B.scan_cloud_msgs(prm, c, 0)
        return ctx.launch_count - k

    plain = [launches(p, d) for d in (False, True)]
    cp.set_transforms(fleet_transforms(rng, n), frames_for(n))
    assert [launches(p, d) for d in (False, True)] == plain
    assert [launches(xf_params(R, SC.params(0x1F)), d) for d in (False, True)] == plain
    cp.close()
    ctx.close()
