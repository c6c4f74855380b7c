"""Projected clouds in a target frame (DESIGN.md 5.7.1 "Projected clouds in a target frame"): laser_geometry's
transformLaserScanToPointCloud with a static transform, restated on the CPU in numpy.  It extends P(params, scan) of
oracle/scan_cloud_oracle.py, which stays the definition of everything not said here; this docstring is the definition
of the transform, and csrc/scan_cloud.cu (scan_cloud_kernel<true>) computes the same bits.

A transform entry is a geometry_msgs/Transform of the published LaserScan frame in the target frame, and a target
frame_id.  It maps a point as p_target = R p_scan + t.

  host, once per entry: R from the quaternion (x, y, z, w) in double, as tf2's Matrix3x3::setRotation:
         d = x^2 + y^2 + z^2 + w^2, s = 2 / d, xs = x s, ys = y s, zs = z s, wx = w xs, wy = w ys, wz = w zs,
         xx = x xs, xy = x ys, xz = x zs, yy = y ys, yz = y zs, zz = z zs,
         R = [[1 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1 - (xx + yy)]];
         each entry is rounded to float once, and so is t (the footprint's rule: the geometry moves once, on the host).
  point: beam i's untransformed point (x_i, y_i, 0) is P's (scan_footprint_oracle.beam_points).  The record's x, y, z
         become, for k = 0, 1, 2, X_k = fl(fl(fl(R_k0 x_i) + fl(R_k1 y_i)) + t_k): no FMA, and no R_k2 term since z is
         0.  An identity transform gives P's records bit for bit for every beam with r_i > 0 (x + 0 = x for x != 0); a
         zero range, kept only by a range_min <= 0, may turn a -0 into +0.
  unchanged: the keep rule, the beam order, intensity, index, distances, stamps, the stamp, height and is_dense.
  frame_id: the entry's target frame.
  viewpoint (VIEWPOINT 0x10): three FLOAT32 fields vp_x, vp_y, vp_z after stamps, each t_k -- the sensor origin in the
         target frame; point_step = 12 + 4 * popcount(channels & 0x0F) + 12 * viewpoint.  The field names and order
         are laser_geometry's as remembered; like the channel names of oracle/scan_cloud_oracle.py they were not
         checked against its source.
  inverted lidars: no special case.  The transform is the pose of the frame the LaserScan is published in, and that
         frame is already mirrored.
  disabled entry (enabled 0): exactly P -- the LaserScan's frame, no transform; the viewpoint fields are 0, 0, 0 (the
         origin in the scan's own frame).  Its transform and frame are not read.
  limits: every value finite, |d - 1| <= 1e-3, |t_k| <= 1000 m, the target frame_id at most 255 characters.  Anything
         else is refused (RPL_RESULT_INVALID_DATA).

The calls: VIEWPOINT is accepted with PER_STREAM_TRANSFORMS (0x100, an option in rpl_scan_cloud_params.channels that
adds no field) or by the stateless call with a transform; PER_STREAM_TRANSFORMS only by the session projections.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from oracle import scan_cloud_oracle as SC

VIEWPOINT, PER_STREAM_TRANSFORMS = 0x10, 0x100
VIEWPOINT_FIELDS = ("vp_x", "vp_y", "vp_z")
MAX_T, MAX_NORM_ERR, MAX_FRAME = 1000.0, 1e-3, 255


def transform(translation=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), enabled=True):
    """the attributes of rpl_scan_cloud_transform"""
    return SimpleNamespace(translation=tuple(float(v) for v in translation),
                           rotation=tuple(float(v) for v in rotation), enabled=bool(enabled))


def transform_ok(e, frame="") -> bool:
    """the limits of an enabled entry (a disabled entry is not read); frame None: the stateless call's, which has none"""
    if not e.enabled:
        return True
    vals = list(e.translation) + list(e.rotation)
    if not all(np.isfinite(v) for v in vals):
        return False
    x, y, z, w = e.rotation
    if not abs(x * x + y * y + z * z + w * w - 1.0) <= MAX_NORM_ERR:
        return False
    if not all(abs(v) <= MAX_T for v in e.translation):
        return False
    return frame is None or len(frame.encode()) <= MAX_FRAME


def rotation_matrix(q) -> np.ndarray:
    """R of the quaternion (x, y, z, w) in double, tf2's Matrix3x3::setRotation"""
    x, y, z, w = (float(v) for v in q)
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return np.array([[1.0 - (yy + zz), xy - wz, xz + wy],
                     [xy + wz, 1.0 - (xx + zz), yz - wx],
                     [xz - wy, yz + wx, 1.0 - (xx + yy)]])


def transform_rows(q, t):
    """(R, t) as the device uses them: R's first two columns [3, 2] and t [3], each rounded to float32 once"""
    return rotation_matrix(q)[:, :2].astype(np.float32), np.asarray(t, np.float64).astype(np.float32)


def params_ok(p, transformed) -> bool:
    """the channel rules of a call with (transformed) or without a transform"""
    extra = VIEWPOINT if transformed else 0
    return (int(p.channels) & ~(SC.CHANNELS | extra | PER_STREAM_TRANSFORMS)) == 0 and SC.params_ok(
        SC.params(int(p.channels) & SC.CHANNELS, p.range_cutoff))


def fields(channels):
    """[(name, offset, datatype, count)] of a channel set, the viewpoint's three fields last"""
    f = SC.fields(int(channels) & SC.CHANNELS)
    if int(channels) & VIEWPOINT:
        f += [(n, 4 * (len(f) + k), SC.FLOAT32, 1) for k, n in enumerate(VIEWPOINT_FIELDS)]
    return f


def point_step(channels) -> int:
    return SC.point_step(int(channels) & SC.CHANNELS) + (12 if int(channels) & VIEWPOINT else 0)


def transform_points(x, y, R, t):
    """X_k = fl(fl(fl(R_k0 x) + fl(R_k1 y)) + t_k) in float32, for k = 0, 1, 2: [3][n]"""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    return [((R[k, 0] * x).astype(np.float32) + (R[k, 1] * y).astype(np.float32)).astype(np.float32) + t[k]
            for k in range(3)]


def project(p, ranges, intensities, inc, time_increment, range_min, range_max, transform=None) -> np.ndarray:
    """the records of P with `transform` (None: P's, the viewpoint refused): [width, point_step] uint8"""
    ch = int(p.channels)
    assert params_ok(p, transform is not None)
    base = SC.params(ch & SC.CHANNELS, p.range_cutoff)
    rec = SC.project(base, ranges, intensities, inc, time_increment, range_min, range_max)
    n = rec.shape[0]
    words = rec.view("<u4").reshape(n, SC.point_step(ch & SC.CHANNELS) // 4).copy()
    on = transform is not None and transform.enabled
    if on:
        R, t = transform_rows(transform.rotation, transform.translation)
        X = transform_points(words[:, 0].view(np.float32), words[:, 1].view(np.float32), R, t)
        for k in range(3):
            words[:, k] = X[k].astype(np.float32).view(np.uint32)
    if ch & VIEWPOINT:
        vp = transform_rows(transform.rotation, transform.translation)[1] if on else np.zeros(3, np.float32)
        words = np.concatenate([words, np.tile(vp.view(np.uint32), (n, 1))], axis=1)
    return np.ascontiguousarray(words.astype("<u4")).view(np.uint8).reshape(n, point_step(ch))


def P(p, scan: dict, transform=None, frame=None) -> bytes:
    """the PointCloud2 message of one LaserScan message with `transform` and its target frame (a disabled entry, or
    None: the scan's frame)"""
    assert float(scan["angle_min"]) == 0.0
    rec = project(p, scan["ranges"], scan["intensities"], scan["angle_increment"], scan["time_increment"],
                  scan["range_min"], scan["range_max"], transform)
    fid = frame if transform is not None and transform.enabled else scan["frame_id"]
    return SC.pointcloud2_fields_cdr(scan["sec"], scan["nanosec"], fid, fields(p.channels), point_step(p.channels),
                                     rec, rec.shape[0])


def project_rows(p, ranges, intensities, beam_counts, angle_increment, time_increment, range_min, range_max,
                 transform=None):
    """P over padded rows [n, stride] (rpl_scan_cloud_transform_batch_dev): ([records per row], kept counts)"""
    out, counts = [], []
    for s in range(ranges.shape[0]):
        M = int(beam_counts[s])
        ti = 0.0 if time_increment is None else time_increment[s]
        rec = project(p, ranges[s, :M], intensities[s, :M], angle_increment[s], ti, range_min, range_max, transform)
        out.append(rec)
        counts.append(rec.shape[0])
    return out, np.asarray(counts, np.uint32)

