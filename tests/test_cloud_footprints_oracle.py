"""Footprints in the clouds (DESIGN.md 5.7.1 "Footprints in the clouds"; RPL_CLOUD_PER_STREAM_FOOTPRINTS and
rpl_cloud_footprint_batch_dev).  This docstring and cloud_with_footprint below are the definition; csrc/cloud_footprint.cu
computes the same bits.

The footprint stage runs on the cloud's step-3 points (oracle/cloud_oracle.cpp), after the window and polar -> xyz and
before SOR (step 4) and the voxel grid (step 5).  A point (x, y) is exactly what the cloud would publish without SOR or
a voxel grid: x = fl(r * c_key), y = fl(r * s_key) from the trig table ((float)cos / sin in double of the float
angle_rad of the key).  It is removed when the crossing-number rule of oracle/scan_footprint_oracle.py `inside` puts
it inside a polygon whose invert is 0, or outside one whose invert is non-zero.  SOR and the voxel grid then run
unchanged on the points left.

Equivalently (the form used here): the cloud with a footprint is the cloud without one of the same nodes with every
removed point's node given dist_mm_q2 = 0, which step 1 skips whatever range_min is.

Frames: the vertices (u, v) are those rpl_capsule_stream_set_scan_footprints computes (scan_footprint_oracle
scan_frame: moved into the LaserScan frame once, in double with libm, rounded to float once).  The cloud is not
mirrored for an inverted lidar, the LaserScan is, so a LaserScan-frame point (xs, ys) is the cloud point (x, -y): an
inverted stream's cloud points are tested against (u, -v) (an exact negation, no new rounding).  The stateless call
mirrors nothing: its footprint's pose is the pose of the cloud's frame.
"""
import functools
import math

import numpy as np
import pytest

from oracle import scan_footprint_oracle as FP


@functools.lru_cache(maxsize=1)
def trig_table():
    """float32 (c, s) of every key as the cloud trig table holds them (csrc/cloud.cu cloud_workspace_alloc): libm's
    cos / sin in double of the float angle_rad, rounded to float"""
    deg = (np.arange(65536, dtype=np.float32) * np.float32(90.0)) / np.float32(16384.0)
    rad = (deg.astype(np.float64) * (math.pi / 180.0)).astype(np.float32)
    c = np.array([math.cos(float(a)) for a in rad], np.float32)
    s = np.array([math.sin(float(a)) for a in rad], np.float32)
    return c, s


def trig(keys):
    c, s = trig_table()
    k = np.asarray(keys, np.int64)
    return c[k], s[k]


def node_points(nodes):
    """float32 (x, y) of every node as step 3 forms it"""
    r = nodes["dist_mm_q2"].astype(np.float32) / np.float32(4000.0)
    c, s = trig(nodes["angle_z_q14"])
    return r * c, r * s


def removed_points(fp, x, y, mirror=False):
    """the footprint stage on points (x, y): which it removes; mirror: an inverted stream's cloud"""
    rm = np.zeros(len(x), bool)
    for u, v, inv in FP.scan_frame(fp):
        rm |= FP.inside(u, -v if mirror else v, x, y) != bool(inv)
    return rm


def cloud_with_footprint(O, nodes, params, fp, mirror=False):
    """the definition: the cloud of the nodes with every removed point's node given dist_mm_q2 = 0"""
    nodes = np.array(nodes, copy=True)
    x, y = node_points(nodes)
    nodes["dist_mm_q2"][removed_points(fp, x, y, mirror) & (nodes["dist_mm_q2"] != 0)] = 0
    return O.cloud(nodes, params)


def kept_nodes(O, nodes, params, fp, mirror=False):
    """the stage inside the chain: the nodes step 1 keeps, in order, without the ones the footprint removes"""
    r = nodes["dist_mm_q2"].astype(np.float32) / np.float32(4000.0)
    q = nodes["quality"].astype(np.float32) if params.is_new_protocol else (nodes["quality"] >> 2).astype(np.float32)
    win = (nodes["dist_mm_q2"] != 0) & (r >= np.float32(params.range_min)) & (r <= np.float32(params.range_max)) & \
        (q >= np.float32(params.intensity_min))
    x, y = node_points(nodes)
    return nodes[win & ~removed_points(fp, x, y, mirror)]


def random_scan(O, rng, n, dup_share=0.0):
    nodes = np.zeros(n, O.NODE_DTYPE)
    key = np.sort(rng.integers(0, 65536, n))
    dup = np.nonzero(rng.random(n) < dup_share)[0]
    dup = dup[dup > 0]
    key[dup] = key[dup - 1]
    rng.shuffle(key[: n // 8])  # a few out of order: the chain's stable sort
    nodes["angle_z_q14"] = key
    nodes["dist_mm_q2"] = rng.integers(0, 8 * 4000, n)
    nodes["dist_mm_q2"][rng.random(n) < 0.05] = 0
    nodes["quality"] = rng.integers(0, 256, n)
    return nodes


def random_footprint(rng, n_poly=None):
    polys, inv = [], []
    for _ in range(int(rng.integers(1, 5)) if n_poly is None else n_poly):
        k = int(rng.integers(3, 17))
        cx, cy = rng.uniform(-3, 3, 2)
        ang = np.sort(rng.uniform(0, 2 * math.pi, k))
        rad = rng.uniform(0.3, 2.5, k)
        polys.append([(cx + a * math.cos(t), cy + a * math.sin(t)) for a, t in zip(rad, ang)])
        inv.append(int(rng.random() < 0.15))
    return FP.footprint(polys, inv, pose=tuple(rng.uniform(-0.5, 0.5, 2)) + (float(rng.uniform(-math.pi, math.pi)),))


def nodes_at(O, pts, quality=200):
    """nodes of (angle_deg, r) pairs (keys and dist rounded to the wire's units)"""
    nodes = np.zeros(len(pts), O.NODE_DTYPE)
    for j, (deg, r) in enumerate(pts):
        nodes[j]["angle_z_q14"] = int(round((deg % 360.0) * 16384 / 90.0)) & 0xFFFF
        nodes[j]["dist_mm_q2"] = int(round(r * 4000))
        nodes[j]["quality"] = quality
    return nodes


def prm(O, **kw):
    kw.setdefault("range_min", 0.15)
    kw.setdefault("range_max", 40.0)
    return O.cloud_params(is_new_protocol=1, **kw)


CHAINS = [dict(), dict(sor_k=8, sor_alpha=1.0), dict(voxel_size=0.05), dict(sor_k=4, sor_alpha=0.5, voxel_size=0.2)]


@pytest.mark.parametrize("n", [1, 2, 33, 500, 4096, 8192])
def test_stage_in_the_chain_is_the_zeroed_node_cloud(oracle, n):
    rng = np.random.default_rng(100 + n)
    nodes = random_scan(oracle, rng, n, dup_share=0.02)
    for mirror in (False, True):
        fp = random_footprint(rng)
        for kw in CHAINS:
            p = prm(oracle, **kw)
            got = cloud_with_footprint(oracle, nodes, p, fp, mirror)
            exp = oracle.cloud(kept_nodes(oracle, nodes, p, fp, mirror), p)
            assert got.tobytes() == exp.tobytes(), (mirror, kw)
    # the points of step 3 are what the window-only cloud publishes
    x, y = node_points(nodes)
    p = prm(oracle)
    kept = kept_nodes(oracle, nodes, p, FP.footprint())
    pts = oracle.cloud(kept, p)
    order = np.argsort(kept["angle_z_q14"], kind="stable")
    kx, ky = node_points(kept[order])
    assert pts[:, 0].tobytes() == kx.tobytes() and pts[:, 1].tobytes() == ky.tobytes()


def seg_dist(px, py, ax, ay, bx, by):
    dx, dy = bx - ax, by - ay
    L = dx * dx + dy * dy
    t = np.clip(((px - ax) * dx + (py - ay) * dy) / L if L > 0 else 0.0, 0.0, 1.0)
    return np.hypot(px - (ax + t * dx), py - (ay + t * dy))


def winding_inside(u, v, px, py):
    """float64 winding number != 0"""
    wn = np.zeros(len(px), np.int64)
    n = len(u)
    for k in range(n):
        ax, ay, bx, by = float(u[k - 1]), float(v[k - 1]), float(u[k]), float(v[k])
        cross = (bx - ax) * (py - ay) - (px - ax) * (by - ay)
        wn += ((ay <= py) & (by > py) & (cross > 0)).astype(np.int64)
        wn -= ((ay > py) & (by <= py) & (cross < 0)).astype(np.int64)
    return wn != 0


def test_decisions_match_float64_winding_away_from_edges(oracle):
    rng = np.random.default_rng(7)
    total = near = 0
    for trial in range(40):
        nodes = random_scan(oracle, rng, 2000)
        nodes = nodes[nodes["dist_mm_q2"] != 0]
        fp = random_footprint(rng, n_poly=1)
        (u, v, inv), = FP.scan_frame(fp)
        x, y = node_points(nodes)
        got = removed_points(fp, x, y)
        r = nodes["dist_mm_q2"].astype(np.float64) / 4000.0
        t = nodes["angle_z_q14"].astype(np.float64) * 2 * math.pi / 65536
        px, py = r * np.cos(t), r * np.sin(t)
        ref = winding_inside(u, v, px, py) != bool(inv)
        d = np.min([seg_dist(px, py, float(u[k - 1]), float(v[k - 1]), float(u[k]), float(v[k]))
                    for k in range(len(u))], axis=0)
        # simple polygons only: a self-crossing random polygon has winding and crossing rules disagree
        if not simple(u, v):
            continue
        tol = 1e-6 * np.maximum(r, 1.0)
        far = d > tol
        assert (got[far] == ref[far]).all(), trial
        total += int(far.sum())
        near += int((~far).sum())
    assert total > 10000 and near < total // 1000


def simple(u, v):
    n = len(u)
    segs = [(float(u[k - 1]), float(v[k - 1]), float(u[k]), float(v[k])) for k in range(n)]

    def cross(a, b, c):
        return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
    for i in range(n):
        for j in range(i + 1, n):
            if j == i + 1 or (i == 0 and j == n - 1):
                continue
            a, b = segs[i][:2], segs[i][2:]
            c, d = segs[j][:2], segs[j][2:]
            if cross(a, b, c) * cross(a, b, d) < 0 and cross(c, d, a) * cross(c, d, b) < 0:
                return False
    return True


def dists(cloud):
    return [round(math.hypot(float(p[0]), float(p[1])), 3) for p in cloud]


def test_body_at_a_corner_turned_45_degrees(oracle):
    # base_link body 0.6 x 0.4 m; the lidar at its front-left corner, turned 45 degrees
    body = [(-0.3, -0.2), (0.3, -0.2), (0.3, 0.2), (-0.3, 0.2)]
    fp = FP.footprint([body], pose=(0.3, 0.2, math.pi / 4))
    into = math.degrees(math.atan2(-0.2, -0.3)) - 45.0  # towards the body's centre, in the lidar frame
    nodes = nodes_at(oracle, [(into, 0.2), (into, 5.0), (into + 180.0, 0.3), (into + 10.0, 0.25)])
    got = cloud_with_footprint(oracle, nodes, prm(oracle), fp)
    assert len(got) == 2  # the body's two returns removed, the wall behind and the return ahead kept
    assert dists(got) == [5.0, 0.3]


def test_box(oracle):
    fp = FP.footprint([[(1.0, -0.5), (2.0, -0.5), (2.0, 0.5), (1.0, 0.5)]])
    nodes = nodes_at(oracle, [(0.0, 1.5), (0.0, 2.5), (10.0, 1.5), (30.0, 1.5), (350.0, 1.2)])
    got = cloud_with_footprint(oracle, nodes, prm(oracle), fp)
    assert dists(got) == [2.5, 1.5]  # 0 deg at 2.5 m, 30 deg at 1.5 m


def test_inverted_region_of_interest(oracle):
    roi = [(-2.0, -2.0), (2.0, -2.0), (2.0, 2.0), (-2.0, 2.0)]
    fp = FP.footprint([roi], invert=[1])
    nodes = nodes_at(oracle, [(0.0, 1.0), (45.0, 3.0), (90.0, 1.9), (200.0, 3.0)])
    got = cloud_with_footprint(oracle, nodes, prm(oracle), fp)
    assert dists(got) == [1.0, 1.9]


def test_concave_l(oracle):
    L = [(0.0, 0.0), (2.0, 0.0), (2.0, 1.0), (1.0, 1.0), (1.0, 2.0), (0.0, 2.0)]
    fp = FP.footprint([L], pose=(-0.5, -0.5, 0.0))  # the lidar at (-0.5, -0.5) in the footprint frame
    # in the lidar frame the notch (1..2, 1..2) is at (1.5..2.5, 1.5..2.5); an arm point at (2.0, 1.0)
    pts = [(45.0, math.hypot(2.0, 2.0)), (math.degrees(math.atan2(1.0, 2.0)), math.hypot(2.0, 1.0)),
           (math.degrees(math.atan2(2.0, 1.0)), math.hypot(1.0, 2.0))]
    got = cloud_with_footprint(oracle, nodes_at(oracle, pts), prm(oracle), fp)
    assert len(got) == 1 and abs(float(got[0, 0]) - 2.0) < 1e-3 and abs(float(got[0, 1]) - 2.0) < 1e-3


def test_polygon_across_angle_zero(oracle):
    tri = [(1.0, -1.0), (3.0, 0.0), (1.0, 1.0)]
    fp = FP.footprint([tri])
    nodes = nodes_at(oracle, [(0.5, 1.5), (359.5, 1.5), (0.0, 1.5), (90.0, 1.5), (180.0, 1.5)])
    got = cloud_with_footprint(oracle, nodes, prm(oracle), fp)
    assert len(got) == 2 and (got[:, 0] < 0.1).all()


def test_inverted_lidar_removes_the_same_body(oracle):
    # the body lies at +y in the LaserScan frame of an inverted lidar: at -y in its (unmirrored) cloud
    body = [(-0.25, 0.5), (0.25, 0.5), (0.25, 1.0), (-0.25, 1.0)]
    fp = FP.footprint([body], pose=(0.0, 0.0, 0.3))
    yaw = 0.3
    c, s = math.cos(yaw), math.sin(yaw)
    bx, by = c * 0.0 + s * 0.75, -s * 0.0 + c * 0.75  # the body's centre in the scan frame
    deg_scan = math.degrees(math.atan2(by, bx))
    r = math.hypot(bx, by)
    nodes = nodes_at(oracle, [(-deg_scan, r), (deg_scan, r)])  # cloud angle of the body: mirrored
    got = cloud_with_footprint(oracle, nodes, prm(oracle), fp, mirror=True)
    assert len(got) == 1 and float(got[0, 1]) > 0  # the body's return gone, the one at +y in the cloud kept
    plain = cloud_with_footprint(oracle, nodes, prm(oracle), fp, mirror=False)
    assert len(plain) == 1 and float(plain[0, 1]) < 0
    # mirroring equals the mirrored footprint, vertices (x, -y) at pose (px, -py, -yaw), bit for bit
    mir = FP.footprint([[(x, -y) for x, y in body]], pose=(0.0, 0.0, -0.3))
    for (u, v, _), (mu, mv, _) in zip(FP.scan_frame(fp), FP.scan_frame(mir)):
        assert u.tobytes() == mu.tobytes() and (-v).tobytes() == mv.tobytes()
    rng = np.random.default_rng(3)
    nodes = random_scan(oracle, rng, 3000)
    for kw in CHAINS:
        p = prm(oracle, **kw)
        assert cloud_with_footprint(oracle, nodes, p, fp, True).tobytes() == \
            cloud_with_footprint(oracle, nodes, p, mir, False).tobytes()


def test_a_removal_changes_a_neighbours_sor_decision(oracle):
    rng = np.random.default_rng(11)
    changed = 0
    for _ in range(20):
        nodes = random_scan(oracle, rng, 600)
        fp = random_footprint(rng)
        p = prm(oracle, sor_k=4, sor_alpha=0.5)
        with_fp = {tuple(q) for q in cloud_with_footprint(oracle, nodes, p, fp)[:, :2].tolist()}
        x, y = node_points(nodes)
        without = oracle.cloud(nodes, p)
        outside = ~removed_points(fp, without[:, 0], without[:, 1])
        after = {tuple(q) for q in without[outside][:, :2].tolist()}
        changed += with_fp != after  # filtering after SOR is not the stage before it
    assert changed > 0


def test_voxel_cell_across_an_edge(oracle):
    fp = FP.footprint([[(2.5, -0.5), (3.5, -0.5), (3.5, 0.5), (2.5, 0.5)]])
    rs = [2.1, 2.2, 2.3, 2.6, 2.7, 2.9]
    nodes = nodes_at(oracle, [(0.0, r) for r in rs])
    got = cloud_with_footprint(oracle, nodes, prm(oracle, voxel_size=1.0), fp)
    assert len(got) == 1 and float(got[0, 0]) < 2.5  # the cell (2, 0)'s centroid of its three outside points
    ref = oracle.cloud(nodes_at(oracle, [(0.0, r) for r in rs[:3]]), prm(oracle, voxel_size=1.0))
    assert got.tobytes() == ref.tobytes()
    assert len(oracle.cloud(nodes, prm(oracle, voxel_size=1.0))) == 1
