"""CPU checks of the re-gridded LaserScan's definition, oracle/rescan_oracle.py: atan2_f64 against libm, the range rule
against hypot, the grid's edges, the seeds and the height band, and Q against a plain float64 re-implementation."""
import math

import numpy as np

from oracle import cdr_oracle as CDR
from oracle import rescan_oracle as RQ
from oracle import scan_cloud_oracle as SC


def _ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-(2**63)) - ia, ia)
    ib = np.where(ib < 0, np.int64(-(2**63)) - ib, ib)
    return np.abs(ia - ib)


def test_atan2_within_one_ulp_of_libm():
    rng = np.random.default_rng(1)
    n = 100_000
    y = rng.normal(size=n) * 10.0 ** rng.uniform(-40, 40, n)
    x = rng.normal(size=n) * 10.0 ** rng.uniform(-40, 40, n)
    # the axes, the diagonals, tiny and huge ratios, every quadrant
    v = np.array([0.0, -0.0, 1.0, -1.0, 1e-300, -1e-300, 1e300, -1e300, 2.0**-29, 0.4375, 0.6875, 1.1875, 2.4375,
                  2.0**66, 3.5, -7.25])
    Y, X = np.meshgrid(v, v)
    y = np.concatenate([y, Y.ravel(), x[:1000] * 1e-20, x[:1000]])
    x = np.concatenate([x, X.ravel(), x[1000:2000], x[1000:2000] * 1e-20])
    got = RQ.atan2_f64(y, x)
    want = np.array([math.atan2(a, b) for a, b in zip(y.tolist(), x.tolist())])
    assert _ulps(got, want).max() <= 1
    assert (np.signbit(got) == np.signbit(want)).all()
    assert RQ.atan_f64(0.5) == math.atan(0.5) or _ulps(RQ.atan_f64(0.5), math.atan(0.5)) <= 1


def test_atan2_special_cases_equal_libm():
    sp = [0.0, -0.0, math.inf, -math.inf, 1.0, -1.0, 2.5, -2.5, 5e-324]
    for y in sp:
        for x in sp:
            if not any(v == 0 or math.isinf(v) for v in (y, x)):
                continue  # not a special case: within 1 ulp, above
            g, e = float(RQ.atan2_f64(y, x)), math.atan2(y, x)
            assert g == e and math.copysign(1, g) == math.copysign(1, e), (y, x, g, e)
    assert math.isnan(RQ.atan2_f64(math.nan, 1.0)) and math.isnan(RQ.atan2_f64(1.0, math.nan))


def test_range_rule_within_one_ulp_of_hypot():
    rng = np.random.default_rng(2)
    x = (rng.normal(size=50_000) * 10.0 ** rng.uniform(-6, 6, 50_000)).astype(np.float32)
    y = (rng.normal(size=50_000) * 10.0 ** rng.uniform(-6, 6, 50_000)).astype(np.float32)
    got = RQ.range_f64(x, y)
    want = np.array([math.hypot(a, b) for a, b in zip(x.astype(np.float64).tolist(), y.astype(np.float64).tolist())])
    assert _ulps(got, want).max() <= 1


def test_ranges_size_and_limits():
    s = RQ.settings()
    assert RQ.ranges_size(s) == 360 and RQ.settings_ok(s)
    assert RQ.ranges_size(RQ.settings(0.0, 1.0, 1.0)) == 1
    assert RQ.ranges_size(RQ.settings(0.0, 1.0, 0.3)) == 4
    assert RQ.ranges_size(RQ.settings(0.0, 8192.0, 1.0)) == 8192
    assert RQ.ranges_size(RQ.settings(0.0, 8193.0, 1.0)) == 0
    bad = [dict(angle_increment=0.0), dict(angle_min=1.0, angle_max=1.0), dict(angle_max=math.nan),
           dict(range_min=-0.1), dict(range_min=5.0, range_max=4.0), dict(min_height=1.0, max_height=0.5),
           dict(inf_epsilon=-1.0), dict(scan_time=math.inf), dict(angle_increment=1e-4)]
    for b in bad:
        assert not RQ.settings_ok(RQ.settings(**b)), b


def test_index_edges():
    """a point exactly at angle_max, points on bin boundaries, and index == ranges_size skipped"""
    s = RQ.settings(0.0, 1.0, 0.25, range_max=100.0)  # 4 bins: [0, .25), [.25, .5), [.5, .75), [.75, 1]
    assert RQ.ranges_size(s) == 4
    a = np.array([0.0, 0.25, 0.5, 0.75, 1.0])
    x, y = (2.0 * np.cos(a)).astype(np.float32), (2.0 * np.sin(a)).astype(np.float32)
    ang = RQ.atan2_f64(y.astype(np.float64), x.astype(np.float64))
    r = RQ.regrid(s, x, y, np.zeros(5, np.float32))
    idx = ((ang - 0.0) / 0.25).astype(np.int64)
    for k in range(4):
        hit = [j for j in range(5) if idx[j] == k and ang[j] <= 1.0]
        assert (r[k] == np.float32(np.inf)) == (not hit)
    # angle_max = 1.0 with an increment that divides it: index 4 == ranges_size is skipped
    s2 = RQ.settings(0.0, 0.5, 0.125, range_max=100.0)
    assert RQ.ranges_size(s2) == 4
    for t in np.linspace(0.49, 0.51, 401):
        x1, y1 = np.float32(np.cos(t)), np.float32(np.sin(t))
        a1 = float(RQ.atan2_f64(float(y1), float(x1)))
        r1 = RQ.regrid(s2, [x1], [y1], [0.0])
        if a1 > 0.5:
            assert np.isinf(r1).all()
        elif int(a1 / 0.125) >= 4:
            assert np.isinf(r1).all()
        else:
            assert np.isfinite(r1).sum() == 1


def test_seeds_and_height_band():
    x, y, z = np.float32([1.0, 2.0, 3.0]), np.float32([0.0, 0.0, 0.0]), np.float32([-1.0, 0.0, 1.0])
    s = RQ.settings(-1.0, 1.0, 0.5, range_max=10.0, min_height=-0.5, max_height=0.5)
    r = RQ.regrid(s, x, y, z)
    assert r[2] == np.float32(2.0) and np.isinf(np.delete(r, 2)).all()
    s = RQ.settings(-1.0, 1.0, 0.5, range_max=10.0, min_height=-1.0, max_height=1.0, use_inf=False, inf_epsilon=0.5)
    r = RQ.regrid(s, x, y, z)
    assert r[2] == np.float32(1.0) and (np.delete(r, 2) == np.float32(10.5)).all()
    s = RQ.settings(-1.0, 1.0, 0.5, range_max=10.0, use_inf=False, inf_epsilon=0.0)
    assert (RQ.regrid(s, [], [], []) == np.float32(10.0)).all()


def _plain(s, x, y, z):
    """a float64 re-implementation with numpy's hypot and arctan2"""
    n = RQ.ranges_size(s)
    out = np.full(n, RQ.seed(s), np.float64)
    for X, Y, Z in zip(x.tolist(), y.tolist(), z.tolist()):
        if Z > s.max_height or Z < s.min_height:
            continue
        r = math.hypot(X, Y)
        if r < s.range_min or r > s.range_max:
            continue
        a = math.atan2(Y, X)
        if a < s.angle_min or a > s.angle_max:
            continue
        i = int((a - s.angle_min) / s.angle_increment)
        if i < n and r < out[i]:
            out[i] = r
    return out.astype(np.float32)


def test_q_against_float64_on_random_clouds():
    rng = np.random.default_rng(3)
    for t in range(30):
        n = int(rng.integers(0, 3000))
        x, y, z = (rng.normal(size=(3, n)) * [[8.0], [8.0], [0.3]]).astype(np.float32)
        lo = float(rng.uniform(-math.pi, 0))
        s = RQ.settings(lo, float(rng.uniform(lo + 0.1, math.pi)), float(rng.uniform(0.001, 0.05)),
                        range_min=float(rng.uniform(0, 1)), range_max=float(rng.uniform(5, 30)),
                        min_height=-0.2, max_height=0.25, use_inf=t % 2 == 0, inf_epsilon=float(rng.uniform(0, 2)))
        got = RQ.regrid(s, x, y, z)
        want = _plain(s, x, y, z)
        diff = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
        if diff.size:  # only where a point lies within 1e-12 rad of a bin edge
            a = np.arctan2(y.astype(np.float64), x.astype(np.float64))
            q = (a - s.angle_min) / s.angle_increment
            edge = np.abs(q - np.round(q)) * s.angle_increment < 1e-12
            near = set(np.floor(q[edge]).astype(int).tolist()) | set(np.round(q[edge]).astype(int).tolist())
            assert set(diff.tolist()) <= near, (t, diff)


def test_q_message_empty_cloud_and_disabled_entry():
    s = RQ.settings(-1.0, 1.0, 0.01, range_max=20.0, use_inf=False, inf_epsilon=1.0, scan_time=0.1)
    cloud = CDR.parse_pointcloud2(SC.pointcloud2_fields_cdr(5, 6, "base_link", SC.fields(0), 12,
                                                            np.zeros((0, 12), np.uint8), 0))
    m = CDR.parse_laserscan(RQ.Q(s, cloud))
    assert (m["sec"], m["nanosec"], m["frame_id"]) == (5, 6, "base_link")
    assert m["ranges"].shape == (RQ.ranges_size(s),) and (m["ranges"] == np.float32(21.0)).all()
    assert m["intensities"].shape == (0,) and m["time_increment"] == 0 and m["scan_time"] == np.float32(0.1)
    assert (m["angle_min"], m["angle_max"], m["angle_increment"]) == (np.float32(-1), np.float32(1), np.float32(0.01))
    assert RQ.Q(RQ.settings(enabled=False), cloud) is None
