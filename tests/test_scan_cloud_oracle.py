"""The restatement of the scan projection, oracle/scan_cloud_oracle.py, against independent statements: float64
trigonometry for the points, hand-built scans for the keep rule, the PointField layout of every channel set, the
footprint stage's own points, and the CDR parser for the message."""
import math

import numpy as np
import pytest

from oracle import cdr_oracle as CDR
from oracle import scan_cloud_oracle as SC
from oracle import scan_footprint_oracle as FP

NAN, INF = float("nan"), float("inf")


def _scan(r, inc=0.01, ti=1e-4, rmin=0.15, rmax=40.0, it=None, sec=12, frame="laser"):
    r = np.asarray(r, np.float32)
    it = np.arange(r.shape[0], dtype=np.float32) if it is None else np.asarray(it, np.float32)
    m = CDR.laserscan_cdr(sec, 34, frame, (0.0, 2 * math.pi, inc, ti, 0.1, rmin, rmax), r, it)
    return CDR.parse_laserscan(m)


def _records(p, scan):
    return SC.cloud_records(CDR.parse_pointcloud2(SC.P(p, scan)))


def _incs(M, mode_a):
    return np.float32(2 * math.pi / (M if mode_a else max(M - 1, 1)))


@pytest.mark.parametrize("mode_a,inv", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_points_against_float64(mode_a, inv):
    rng = np.random.default_rng(3 + 2 * mode_a + inv)
    for M in (1, 2, 3, 17, 360, 1000, 3200, 4095, 4096, 8191, 8192):
        inc = _incs(M, mode_a)
        r = rng.uniform(0.15, 39.0, M).astype(np.float32)
        if inv:  # an inverted scan is the reversed one: its beam grid is the same
            r = r[::-1].copy()
        if mode_a:
            r[rng.random(M) < 0.1] = np.inf
        rec = _records(SC.params(SC.CHANNELS), _scan(r, inc=inc))
        i = rec["index"].astype(np.int64)
        a = i.astype(np.float64) * np.float64(inc)
        rr = r[i].astype(np.float64)
        tol = 1e-6 * rr
        assert (np.abs(rec["x"] - rr * np.cos(a)) <= tol).all(), M
        assert (np.abs(rec["y"] - rr * np.sin(a)) <= tol).all(), M
        assert (rec["z"] == 0).all()
        assert i.tolist() == np.flatnonzero(np.isfinite(r) & (r >= np.float32(0.15)) & (r < np.float32(40))).tolist()


def test_points_are_the_footprint_stage_points():
    rng = np.random.default_rng(5)
    for M in (1, 7, 4096, 8192):
        inc = _incs(M, M % 2)
        r = rng.uniform(0.2, 30.0, M).astype(np.float32)
        x, y = FP.beam_points(r, inc)
        rec = _records(SC.params(SC.INDEX | SC.DISTANCE), _scan(r, inc=inc))
        assert rec["x"].tobytes() == x.tobytes() and rec["y"].tobytes() == y.tobytes()
        assert rec["distances"].tobytes() == r.tobytes()


def test_keep_rule_on_hand_built_scans():
    r = [NAN, INF, -INF, 0.15, np.nextafter(np.float32(0.15), np.float32(0)), 5.0, 40.0,
         np.nextafter(np.float32(40.0), np.float32(0)), 1e6, 0.0]
    keep = lambda p, **kw: _records(p, _scan(r, **kw))["index"].tolist()  # noqa: E731
    assert keep(SC.params(SC.INDEX)) == [3, 5, 7]                         # range_min <= r < range_max
    assert keep(SC.params(SC.INDEX, -1.0)) == keep(SC.params(SC.INDEX, -1e-30)) == [3, 5, 7]
    assert keep(SC.params(SC.INDEX, 5.0)) == [3]                          # r == cutoff is not kept
    assert keep(SC.params(SC.INDEX, 1e7)) == [3, 5, 6, 7, 8]              # a cutoff above range_max
    assert keep(SC.params(SC.INDEX, INF)) == [3, 5, 6, 7, 8]              # +inf is never kept
    assert keep(SC.params(SC.INDEX, 0.0)) == []
    assert keep(SC.params(SC.INDEX), rmin=0.0) == [3, 4, 5, 7, 9]
    assert keep(SC.params(SC.INDEX), rmax=1e30) == [3, 5, 6, 7, 8]


def test_every_channel_set_layout():
    r = np.array([1.0, NAN, 2.0, 3.0], np.float32)
    names = ["intensity", "index", "distances", "stamps"]
    types = [SC.FLOAT32, SC.INT32, SC.FLOAT32, SC.FLOAT32]
    for ch in range(16):
        p = SC.params(ch)
        msg = CDR.parse_pointcloud2(SC.P(p, _scan(r, ti=2.5e-4, frame="abc")))
        present = [k for k in range(4) if ch >> k & 1]
        want = [("x", 0, SC.FLOAT32, 1), ("y", 4, SC.FLOAT32, 1), ("z", 8, SC.FLOAT32, 1)] + \
            [(names[k], 12 + 4 * j, types[k], 1) for j, k in enumerate(present)]
        assert msg["fields"] == want
        assert msg["point_step"] == 12 + 4 * len(present) == SC.point_step(ch)
        assert msg["height"] == 1 and msg["width"] == 3 and msg["row_step"] == 3 * msg["point_step"]
        assert msg["is_bigendian"] == 0 and msg["is_dense"] == 1
        assert (msg["sec"], msg["nanosec"], msg["frame_id"]) == (12, 34, "abc")
        rec = SC.cloud_records(msg)
        if ch & SC.INTENSITY:
            assert rec["intensity"].tolist() == [0.0, 2.0, 3.0]
        if ch & SC.INDEX:
            assert rec["index"].tolist() == [0, 2, 3]
        if ch & SC.TIMESTAMP:
            assert rec["stamps"].tobytes() == (np.float32([0, 2, 3]) * np.float32(2.5e-4)).tobytes()


def test_field_list_writer_is_the_node_cloud_writer_for_its_fields():
    """the general writer with the node cloud's fields gives cdr_oracle.pointcloud2_cdr's bytes"""
    rng = np.random.default_rng(13)
    fields = [(n, 4 * k, SC.FLOAT32, 1) for k, n in enumerate(("x", "y", "z", "intensity"))]
    for n, frame in ((0, ""), (1, "a"), (5, "abcd"), (300, "laser_frame")):
        xyzi = rng.uniform(-9, 9, (n, 4)).astype(np.float32)
        got = SC.pointcloud2_fields_cdr(7, 8, frame, fields, 16, xyzi, n)
        assert got == CDR.pointcloud2_cdr(7, 8, frame, xyzi)
        rec = SC.cloud_records(CDR.parse_pointcloud2(got))
        assert rec["intensity"].tobytes() == np.ascontiguousarray(xyzi[:, 3]).tobytes()


def test_params_rules():
    assert all(SC.params_ok(SC.params(ch, c)) for ch in range(16) for c in (-1.0, 0.0, 3.0, INF, -INF))
    assert not SC.params_ok(SC.params(0x10)) and not SC.params_ok(SC.params(0x1F))
    assert not SC.params_ok(SC.params(0x03, NAN))


def test_empty_scan_gives_width_zero():
    msg = CDR.parse_pointcloud2(SC.P(SC.params(), _scan([NAN, INF, 0.01])))
    assert msg["width"] == 0 and msg["row_step"] == 0 and msg["data"].size == 0


def test_footprinted_scan_projects_no_removed_point():
    rng = np.random.default_rng(11)
    box = [(-2.0, -1.0), (2.0, -1.0), (2.0, 1.0), (-2.0, 1.0)]
    fp = FP.footprint([box], pose=(0.5, 0.2, 0.4))
    for M in (360, 3200, 8192):
        inc = _incs(M, 0)
        r = rng.uniform(0.15, 6.0, M).astype(np.float32)
        removed = FP.removed_footprint(fp, r, inc)
        assert removed.any()
        rf = r.copy()
        rf[removed] = np.float32(np.nan)
        rec = _records(SC.params(SC.INDEX), _scan(rf, inc=inc))
        assert not removed[rec["index"]].any()
        x, y = rec["x"], rec["y"]
        for u, v, inv in FP.scan_frame(fp):
            assert not (FP.inside(u, v, x, y) != bool(inv)).any()
        assert rec.shape[0] == int((~removed).sum())
