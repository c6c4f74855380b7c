"""CPU checks of the footprint stage's definition (oracle/scan_footprint_oracle.py): the beam directions against numpy
over every angle a scan can have, the float32 restatement's decisions against an independent float64 point-in-polygon
test, hand-built scans of the filters it stands for, and its limits."""
import math

import numpy as np
import pytest

from oracle import scan_filter_oracle as F
from oracle import scan_footprint_oracle as FP

INC360 = np.float32(2 * math.pi / 360)


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _removed(out):
    return np.flatnonzero(np.isnan(out))


def _run(fp, r, inc=INC360, s=None, it=None):
    r = np.asarray(r, np.float32)
    it = np.ones(r.shape[0], np.float32) if it is None else it
    return FP.filter_scan(F.settings() if s is None else s, fp, r, it, inc)


def _ulps(g, e):
    """float32 ulp distance, a sign change at a zero crossing compared by value"""
    d = np.abs(g.view(np.int32).astype(np.int64) - e.view(np.int32).astype(np.int64))
    return np.where(np.signbit(g) == np.signbit(e), d, (np.abs(g - e) > np.spacing(np.float32(1e-30))) * 2)


def test_beam_directions_within_one_ulp_for_every_beam_count():
    """(s_i, c_i) of every i * inc, i < M, Mode A (inc = fl(2 pi / M)) and Mode B (fl(2 pi / (M - 1))), M in [2, 8192]"""
    for lo in range(2, 8193, 512):
        M = np.arange(lo, min(lo + 512, 8193))
        for inc in ((2 * np.pi / M).astype(np.float32), (2 * np.pi / (M - 1)).astype(np.float32)):
            i = np.concatenate([np.arange(m) for m in M]).astype(np.float64)
            x = i * np.repeat(inc.astype(np.float64), M)
            s, c = FP.SF.sincos_f64(x)
            assert (_ulps(s.astype(np.float32), np.sin(x).astype(np.float32)) <= 1).all()
            assert (_ulps(c.astype(np.float32), np.cos(x).astype(np.float32)) <= 1).all()


# ---- the restatement against an independent float64 statement ----------------------------------------------------
def _f64_removed(fp, r, inc):
    """(removed, distance to the nearest polygon boundary) in float64: the points and the polygons both in the
    footprint frame, inside by the winding number"""
    M = r.shape[0]
    th = np.arange(M) * float(inc)
    c, s = math.cos(fp.pose_yaw), math.sin(fp.pose_yaw)
    fin = np.isfinite(r)
    rr = np.where(fin, r, 0).astype(np.float64)
    lx, ly = rr * np.cos(th), rr * np.sin(th)
    X, Y = fp.pose_x + c * lx - s * ly, fp.pose_y + s * lx + c * ly
    rm, dist = np.zeros(M, bool), np.full(M, np.inf)
    for p in range(4):
        n = fp.n_vertices[p]
        if n == 0:
            continue
        vx, vy = fp.x[p][:n].astype(np.float64), fp.y[p][:n].astype(np.float64)
        wind = np.zeros(M, np.int64)
        for k in range(n):
            ax, ay, bx, by = vx[k - 1], vy[k - 1], vx[k], vy[k]
            cross = (bx - ax) * (Y - ay) - (X - ax) * (by - ay)
            wind += ((ay <= Y) & (by > Y) & (cross > 0)).astype(np.int64)
            wind -= ((ay > Y) & (by <= Y) & (cross < 0)).astype(np.int64)
            ex, ey = bx - ax, by - ay
            t = np.clip(((X - ax) * ex + (Y - ay) * ey) / (ex * ex + ey * ey), 0, 1)
            dist = np.minimum(dist, np.hypot(X - ax - t * ex, Y - ay - t * ey))
        rm |= (wind != 0) != bool(fp.invert[p])
    return rm & fin, dist


def _star(rng, n, cx, cy, rmin, rmax):
    """a simple polygon of n vertices, star-shaped about (cx, cy) (concave in general)"""
    a = np.sort(rng.uniform(0, 2 * math.pi, n))
    rad = rng.uniform(rmin, rmax, n)
    return [(float(cx + q * math.cos(t)), float(cy + q * math.sin(t))) for t, q in zip(a, rad)]


def _random_footprint(rng):
    k = int(rng.integers(1, 5))
    polys = [_star(rng, int(rng.integers(3, 17)), *rng.uniform(-3, 3, 2), 0.2, 6.0) for _ in range(k)]
    inv = [int(rng.random() < 0.3) for _ in range(k)]
    pose = (*rng.uniform(-2, 2, 2), rng.uniform(-10, 10))
    return FP.footprint(polys, inv, pose)


@pytest.mark.parametrize("seed", range(8))
def test_restatement_against_float64(seed):
    from test_scan_filters_oracle import _random_scan

    rng = np.random.default_rng(seed)
    near, removed, total = 0, 0, 0
    for _ in range(4):
        M = int(rng.integers(2, 8193))
        inc = np.float32(2 * math.pi / (M if rng.random() < 0.5 else M - 1))
        r, _ = _random_scan(rng, M)
        fp = _random_footprint(rng)
        assert FP.footprint_ok(fp)
        got = FP.removed_footprint(fp, r, inc)
        want, dist = _f64_removed(fp, r, inc)
        bad = got != want
        tol = 1e-6 * np.maximum(np.where(np.isfinite(r), r, 0), 1.0)
        assert (dist[bad] < tol[bad]).all()
        near += int(bad.sum())
        removed += int(got.sum())
        total += M
    assert removed > total // 20
    assert near <= max(2, total // 10000)


# ---- hand-built scans -------------------------------------------------------------------------------------------
def test_body_with_the_lidar_at_a_corner():
    """a 1.0 x 0.6 m body about base_link, the lidar on its front-left corner turned 45 degrees: a return off the body
    is removed, the wall behind the body in the same direction is kept, and the angular mask that would hide the body
    would hide the wall too"""
    fp = FP.footprint([[(-0.5, -0.3), (0.5, -0.3), (0.5, 0.3), (-0.5, 0.3)]], pose=(0.5, 0.3, math.radians(45)))
    r = np.full(360, 5.0, np.float32)
    # base_link direction 200 degrees from the corner is scan angle 155 degrees: 0.4 m lands at (0.124, 0.163)
    r[155] = 0.4
    r[0] = 0.4  # ahead of the lidar, away from the body
    out = _run(fp, r)
    assert np.isnan(out[155]) and out[0] == np.float32(0.4)
    assert out[156] == np.float32(5.0) and out[154] == np.float32(5.0)  # the wall behind the body
    want, _ = _f64_removed(fp, r, INC360)
    assert (np.isnan(out) == want).all()
    assert _removed(out).tolist() == [155]


def test_box_filter_as_one_polygon():
    """LaserScanBoxFilter over x, y in [-0.25, 0.25] about the lidar: every point inside the box goes"""
    box = [(-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)]
    M = 720
    inc = np.float32(2 * math.pi / M)
    rng = np.random.default_rng(3)
    r = rng.uniform(0.05, 0.5, M).astype(np.float32)
    out = _run(FP.footprint([box]), r, inc)
    th = np.arange(M) * float(inc)
    x, y = r * np.cos(th), r * np.sin(th)
    inside = (np.abs(x) < 0.25) & (np.abs(y) < 0.25)
    margin = np.minimum(np.abs(np.abs(x) - 0.25), np.abs(np.abs(y) - 0.25))
    clear = margin > 1e-5
    assert (np.isnan(out)[clear] == inside[clear]).all()
    assert inside.sum() > 100 and (~inside).sum() > 100
    assert (_bits(out[~np.isnan(out)]) == _bits(r[~np.isnan(out)])).all()
    # inverted: the box is the region of interest, what lies outside it goes
    out = _run(FP.footprint([box], invert=[1]), r, inc)
    assert (np.isnan(out)[clear] == ~inside[clear]).all()


def test_inverted_region_of_interest():
    """a triangle ahead of the robot as the region of interest, the scan frame 1 m behind base_link"""
    tri = [(0.0, -2.0), (4.0, 0.0), (0.0, 2.0)]
    fp = FP.footprint([tri], invert=[1], pose=(-1.0, 0.0, 0.0))
    r = np.full(360, 1.5, np.float32)
    out = _run(fp, r)
    # beam 0 lands at base_link (0.5, 0): inside, kept; beam 180 at (-2.5, 0): outside, removed
    assert out[0] == np.float32(1.5) and np.isnan(out[180]) and np.isnan(out[90])
    want, _ = _f64_removed(fp, r, INC360)
    assert (np.isnan(out) == want).all()


def test_concave_l_shape():
    L = [(0.0, 0.0), (2.0, 0.0), (2.0, 1.0), (1.0, 1.0), (1.0, 2.0), (0.0, 2.0)]
    fp = FP.footprint([L], pose=(0.0, 0.0, 0.0))
    r = np.full(360, 10.0, np.float32)
    r[45] = 1.2 * math.sqrt(2)   # (1.2, 1.2): in the notch, kept
    r[44] = 1.8                  # ~(1.29, 1.25): in the notch, kept
    r[10] = 1.5                  # (1.48, 0.26): the lower arm, removed
    r[80] = 1.5                  # (0.26, 1.48): the upper arm, removed
    r[30] = 0.8                  # (0.69, 0.4): the corner square, removed
    out = _run(fp, r)
    assert _removed(out).tolist() == [10, 30, 80]
    want, _ = _f64_removed(fp, r, INC360)
    assert (np.isnan(out) == want).all()


def test_polygon_across_angle_zero():
    """a box straddling the scan's x axis: the first and the last beams of the revolution fall in it"""
    fp = FP.footprint([[(1.0, -0.3), (2.0, -0.3), (2.0, 0.3), (1.0, 0.3)]])
    r = np.full(360, 1.5, np.float32)
    out = _run(fp, r)
    rm = _removed(out).tolist()
    # 1.5 m lands inside the box within atan(0.3 / 1.5) = 11.3 degrees of the x axis, on both sides of angle 0
    assert rm == list(range(0, 12)) + list(range(349, 360))
    want, _ = _f64_removed(fp, r, INC360)
    assert (np.isnan(out) == want).all()


def test_non_finite_ranges_untouched():
    """Mode A's +inf bins and an earlier NaN inside an inverted region of interest's outside stay as they are"""
    fp = FP.footprint([[(-1.0, -1.0), (1.0, -1.0), (1.0, 1.0), (-1.0, 1.0)]], invert=[1])
    r = np.full(360, 5.0, np.float32)
    odd_nan = np.array([0x7FC00123], np.uint32).view(np.float32)[0]
    r[[3, 4, 5]] = [np.inf, odd_nan, -np.inf]
    r[100] = 0.5
    out = _run(fp, r)
    assert (_bits(out[[3, 4, 5]]) == _bits(r[[3, 4, 5]])).all()
    assert out[100] == np.float32(0.5)
    assert (_bits(np.delete(out, [3, 4, 5, 100])) == F.NAN_BITS).all()
    # a disabled entry leaves the scan as it is, footprint or not
    s = F.settings(enabled=False)
    assert (_bits(_run(fp, r, s=s)) == _bits(r)).all()


def test_removed_beam_makes_its_neighbour_a_speckle():
    """beams 20 and 21 are a two-beam cluster that the speckle stage keeps; the footprint removes beam 20, so beam 21
    is left without a neighbour and the speckle stage, which runs after it, removes it"""
    r = np.full(360, 5.0, np.float32)
    r[20:22] = 0.5
    th = 20 * float(INC360)
    px, py = 0.5 * math.cos(th), 0.5 * math.sin(th)
    d = 0.003
    fp = FP.footprint([[(px - d, py - d), (px + d, py - d), (px + d, py + d), (px - d, py + d)]])
    s = F.settings(speckle_window=1, speckle_min_neighbours=1, speckle_max_diff=0.05)
    assert _removed(_run(None, r, s=s)).tolist() == []
    assert _removed(FP.filter_scan(F.settings(), fp, r, np.ones(360, np.float32), INC360)).tolist() == [20]
    assert _removed(_run(fp, r, s=s)).tolist() == [20, 21]


def test_no_polygon_is_the_filter_chain():
    from test_scan_filters_oracle import _random_scan, _random_settings

    rng = np.random.default_rng(5)
    for _ in range(4):
        M = int(rng.integers(2, 3000))
        r, it = _random_scan(rng, M)
        s = _random_settings(rng)
        want = F.filter_scan(s, r, it, INC360)
        for fp in (None, FP.footprint(), FP.footprint(pose=(3.0, -2.0, 1.0))):
            assert (_bits(FP.filter_scan(s, fp, r, it, INC360)) == _bits(want)).all()


# ---- limits -----------------------------------------------------------------------------------------------------
TRI = [(0.0, 0.0), (1.0, 0.0), (0.0, 1.0)]
# footprints the library refuses with RPL_RESULT_INVALID_DATA (tests/test_gpu_scan_footprints.py plays them against it)
BAD = [
    dict(polygons=[TRI[:1]]),
    dict(polygons=[TRI[:2]]),
    dict(polygons=[[(float(k), float(k * k)) for k in range(16)]], n_vertices=17),
    dict(polygons=[TRI, [(0.0, 0.0), (math.nan, 0.0), (0.0, 1.0)]]),
    dict(polygons=[[(0.0, 0.0), (math.inf, 0.0), (0.0, 1.0)]]),
    dict(polygons=[[(0.0, 0.0), (1000.5, 0.0), (0.0, 1.0)]]),
    dict(polygons=[[(0.0, -1001.0), (1.0, 0.0), (0.0, 1.0)]]),
    dict(polygons=[TRI], pose=(math.nan, 0.0, 0.0)),
    dict(polygons=[TRI], pose=(0.0, 1000.5, 0.0)),
    dict(polygons=[TRI], pose=(0.0, 0.0, math.inf)),
    dict(pose=(-1001.0, 0.0, 0.0)),
]
GOOD = [
    dict(),
    dict(polygons=[TRI], invert=[1, 1, 1, 1]),
    dict(polygons=[[(1000.0, -1000.0), (1000.0, 1000.0), (-1000.0, 0.0)]], pose=(-1000.0, 1000.0, 100.0)),
    dict(polygons=[[(math.cos(k / 2.5), math.sin(k / 2.5)) for k in range(16)]] * 4),
    dict(polygons=[[], TRI, [], TRI]),
]


def make(build, kw):
    """build(**kw) (FP.footprint or capi.scan_footprint), n_vertices overriding the first polygon's count"""
    kw = dict(kw)
    n = kw.pop("n_vertices", None)
    fp = build(**kw)
    if n is not None:
        fp.n_vertices[0] = n
    return fp


def test_footprint_limits():
    assert not any(FP.footprint_ok(make(FP.footprint, kw)) for kw in BAD)
    assert all(FP.footprint_ok(make(FP.footprint, kw)) for kw in GOOD)
    # vertices past n_vertices, and those of an unused polygon, are not looked at
    fp = FP.footprint([TRI])
    fp.x[0][3:] = np.nan
    fp.y[1][:] = np.inf
    assert FP.footprint_ok(fp)
