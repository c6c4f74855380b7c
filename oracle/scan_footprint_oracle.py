"""The footprint stage of the LaserScan filter chain (DESIGN.md 5.7.1 "LaserScan filters"), restated on the CPU in
numpy float32, and the chain F(settings, footprint, scan) with it.  This docstring and oracle/scan_filter_oracle.py's
are the definition; csrc/scan_filter.cu computes the same bits.

Footprint: up to 4 polygons, each of 3..16 vertices (n_vertices 0: an unused polygon) with an invert bit.  A beam is
removed when its point lies inside a polygon whose invert is 0 (the robot's own body: LaserScanPolygonFilter,
LaserScanBoxFilter), or outside one whose invert is 1 (a region of interest) -- what a chain of laser_filters polygon
filters gives.  The vertices are given in the footprint frame (base_link); (pose_x, pose_y, pose_yaw) is the pose of
the published LaserScan frame (the inversion already applied) in that frame.

The footprint is pointwise: it runs beside stages 1-3 (mask, range window, intensity floor), deciding every beam from
the chain's input, so a beam it removes is already NaN when speckle (4) and veiling (5) look at it -- a laser_filters
chain with the polygon filter first.  Like the other stages it tests finite ranges only, and it changes no
intensity, beam count, increment or message size; a removed range becomes 0x7FC00000.

  frame: each used vertex (vx, vy) is moved into the scan frame once, on the host, in double with every operation
         rounded as written, and rounded to float once:
           c, s = cos(double(pose_yaw)), sin(double(pose_yaw))  (libm: math.cos / math.sin, not numpy's vector trig)
           u = c * (vx - px) + s * (vy - py),  v = -s * (vx - px) + c * (vy - py)
  beam point: for a finite r_i, (s_i, c_i) = float(sincos_f64(double(i) * double(inc))) (scan_filter_oracle's
         sincos_f64; i * inc is exact in double as i < 2^13 and inc is a float), x = fl(r_i * c_i), y = fl(r_i * s_i).
         (The mask stage keeps its float angle fl(i * inc).)
  inside: the crossing-number rule over the edges (v_{k-1}, v_k), k = 0..n-1 (v_{-1} = v_{n-1}): an edge (xa, ya)-(xb, yb)
         is counted when (ya > y) != (yb > y) and x < fl(xa + fl(fl(fl(xb - xa) * fl(y - ya)) / fl(yb - ya))); the
         point is inside when the count is odd.  Every float operation is rounded as written, no FMA; the straddle
         condition leaves out horizontal edges, so the divisor is never 0.  A point exactly on an edge is inside or
         outside as this rule decides.

Limits (footprint_ok): n_vertices 0 or 3..16, every used vertex and the pose finite, |vx|, |vy|, |pose_x|, |pose_y|
<= 1000 (metres).
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

from oracle import scan_filter_oracle as SF

MAX_POLYGONS = 4
MAX_VERTICES = 16
MAX_COORD = 1000.0


def footprint(polygons=(), invert=(), pose=(0.0, 0.0, 0.0)):
    """A footprint with the attributes of rpl_scan_footprint (float32 values, as the struct holds them): polygons is up
    to four vertex lists [(x, y), ...] in the footprint frame, invert their bits (missing: 0), pose (x, y, yaw) of the
    scan frame in the footprint frame."""
    assert len(polygons) <= MAX_POLYGONS and len(invert) <= MAX_POLYGONS
    x = np.zeros((MAX_POLYGONS, MAX_VERTICES), np.float32)
    y = np.zeros((MAX_POLYGONS, MAX_VERTICES), np.float32)
    n = [0] * MAX_POLYGONS
    for p, poly in enumerate(polygons):
        assert len(poly) <= MAX_VERTICES
        n[p] = len(poly)
        for k, (vx, vy) in enumerate(poly):
            x[p, k], y[p, k] = vx, vy
    inv = [int(bool(b)) for b in invert] + [0] * (MAX_POLYGONS - len(invert))
    px, py, pyaw = (float(np.float32(v)) for v in pose)
    return SimpleNamespace(x=x, y=y, n_vertices=n, invert=inv, pose_x=px, pose_y=py, pose_yaw=pyaw)


def footprint_ok(fp) -> bool:
    """The limits rpl_scan_filter_footprint_batch_dev and rpl_capsule_stream_set_scan_footprints enforce."""
    pose = [float(np.float32(v)) for v in (fp.pose_x, fp.pose_y, fp.pose_yaw)]
    if not all(math.isfinite(v) for v in pose) or abs(pose[0]) > MAX_COORD or abs(pose[1]) > MAX_COORD:
        return False
    for p in range(MAX_POLYGONS):
        n = int(fp.n_vertices[p])
        if n == 0:
            continue
        if not 3 <= n <= MAX_VERTICES:
            return False
        v = np.concatenate([np.asarray(fp.x[p][:n], np.float32), np.asarray(fp.y[p][:n], np.float32)])
        if not (np.isfinite(v).all() and (np.abs(v) <= MAX_COORD).all()):
            return False
    return True


def scan_frame(fp):
    """[(u[n], v[n], invert)] of the used polygons, moved into the scan frame (float32)"""
    c, s = math.cos(float(fp.pose_yaw)), math.sin(float(fp.pose_yaw))
    px, py = float(fp.pose_x), float(fp.pose_y)
    out = []
    for p in range(MAX_POLYGONS):
        n = int(fp.n_vertices[p])
        if n == 0:
            continue
        u, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
        for k in range(n):
            dx, dy = float(np.float32(fp.x[p][k])) - px, float(np.float32(fp.y[p][k])) - py
            u[k] = np.float32(c * dx + s * dy)
            v[k] = np.float32(-s * dx + c * dy)
        out.append((u, v, int(bool(fp.invert[p]))))
    return out


def beam_points(r, inc):
    """float32 (x, y) of every beam: x = fl(r_i * c_i), y = fl(r_i * s_i)"""
    r = np.asarray(r, np.float32)
    s, c = SF.sincos_f64(np.arange(r.shape[0], dtype=np.float64) * float(np.float32(inc)))
    with np.errstate(invalid="ignore", over="ignore"):
        return r * c.astype(np.float32), r * s.astype(np.float32)


def inside(u, v, x, y):
    """the crossing-number rule in float32 for points (x, y) against the polygon (u, v)"""
    n = u.shape[0]
    odd = np.zeros(x.shape[0], bool)
    for k in range(n):
        xa, ya, xb, yb = u[k - 1], v[k - 1], u[k], v[k]
        st = (ya > y) != (yb > y)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            xi = xa + ((xb - xa) * (y - ya)) / (yb - ya)
        odd ^= st & (x < xi)
    return odd


def removed_footprint(fp, r, inc):
    """the footprint stage on ranges r: the finite beams it removes"""
    r = np.asarray(r, np.float32)
    rm = np.zeros(r.shape[0], bool)
    polys = scan_frame(fp)
    if not polys:
        return rm
    fin = np.isfinite(r)
    x, y = beam_points(np.where(fin, r, np.float32(0)), inc)
    for u, v, inv in polys:
        rm |= inside(u, v, x, y) != bool(inv)
    return rm & fin


def filter_scan(s, fp, ranges, intensities, inc):
    """F(s, fp, scan): the filtered ranges (float32, same length); fp None: no footprint.  A disabled entry returns the
    ranges as they are, footprint or not."""
    r = np.array(ranges, dtype=np.float32, copy=True)
    if not s.enabled or r.shape[0] == 0:
        return r
    with np.errstate(invalid="ignore", over="ignore"):
        rm = SF.removed_pointwise(s, r, intensities, inc)
        if fp is not None:
            rm |= removed_footprint(fp, r, inc)
        r[rm] = SF._nan()
        if s.speckle_window > 0:
            r[SF.removed_speckle(s, r)] = SF._nan()
        if s.shadow_window > 0:
            r[SF.removed_veiling(s, r, inc)] = SF._nan()
    return r


def filter_rows(entries, footprints, ranges, intensities, beam_counts, angle_increment, per=None):
    """F over padded rows [n, stride]: row s takes entries[s // per] and footprints[s // per] (per None: the one entry
    and footprint for every row; footprints None: none).  Returns the filtered copy of ranges."""
    out = np.array(ranges, dtype=np.float32, copy=True)
    for s in range(out.shape[0]):
        e = entries if per is None else entries[s // per]
        fp = footprints if per is None or footprints is None else footprints[s // per]
        M = int(beam_counts[s])
        if M:
            out[s, :M] = filter_scan(e, fp, out[s, :M], intensities[s, :M], angle_increment[s])
    return out
