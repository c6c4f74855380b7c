"""The projection of a published LaserScan into a PointCloud2 (DESIGN.md 5.7.1 "Clouds projected from the LaserScans"),
laser_geometry's LaserProjection::projectLaser, restated on the CPU in numpy float32.  This docstring is the
definition; csrc/scan_cloud.cu computes the same bits.

P(params, scan) is a pure function of one published LaserScan: its ranges r_i, intensities, angle_increment inc,
time_increment, range_min and range_max.  angle_min is 0, and the scan mode and the inversion are already applied
(the filters and footprints too, when the scan had them).

  beam point: x_i = fl(r_i * c_i), y_i = fl(r_i * s_i), z = 0, where (s_i, c_i) are the float-rounded
         sincos_f64(double(i) * double(inc)): scan_footprint_oracle.beam_points, bit for bit -- a projected point is
         exactly the point the footprint stage of the filters tested.
  kept:  beam i is kept iff range_min <= r_i < cutoff, cutoff = params.range_cutoff when that is >= 0, else the scan's
         range_max (float32 comparisons).  NaN (a filtered beam) and +inf (a Mode A bin without a node) are never
         kept.  The kept beams appear in beam order.
  channels (the bits of laser_geometry's ChannelOption; the default 0x03):
           INTENSITY 0x01  intensity  FLOAT32  intensities[i]
           INDEX     0x02  index      INT32    i
           DISTANCE  0x04  distances  FLOAT32  r_i
           TIMESTAMP 0x08  stamps     FLOAT32  fl(float(i) * time_increment)
         The fields x, y, z (FLOAT32) come first, then the present channels in this order, each 4 bytes at offsets
         0, 4, 8, ...; point_step = 12 + 4 * popcount(channels).  Any other bit is refused, VIEWPOINT 0x10 included
         (its fields are constant zeros).
  message: the LaserScan's header (stamp, frame_id); height 1, width the kept count, is_bigendian 0, row_step =
         point_step * width, is_dense 1 (every kept point is finite; the value of oracle/cdr_oracle.py
         pointcloud2_cdr -- laser_geometry's own value was not checked).

The field names and the cutoff rule are laser_geometry's as remembered: its source was not at hand when this was
written, so this restatement's bytes are the definition either way.  high_fidelity (per-point motion) and target
frames are not served.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from oracle import cdr_oracle as CDR
from oracle import scan_footprint_oracle as SFP

# PointField datatypes
INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
_FIELD_FMT = {INT8: "i1", UINT8: "u1", INT16: "<i2", UINT16: "<u2", INT32: "<i4", UINT32: "<u4", FLOAT32: "<f4",
              FLOAT64: "<f8"}

INTENSITY, INDEX, DISTANCE, TIMESTAMP = 0x01, 0x02, 0x04, 0x08
CHANNELS = 0x0F
DEFAULT = INTENSITY | INDEX
# (bit, field name, datatype) in field order
CHANNEL_FIELDS = ((INTENSITY, "intensity", FLOAT32), (INDEX, "index", INT32),
                  (DISTANCE, "distances", FLOAT32), (TIMESTAMP, "stamps", FLOAT32))


def pointcloud2_fields_cdr(sec, nanosec, frame_id, fields, point_step, data, width, is_dense=1) -> bytes:
    """An unorganised PointCloud2 (height 1) of any field list, by cdr_oracle's CDR rules: fields [(name, offset,
    datatype, count)], data the width * point_step bytes of the points.  (cdr_oracle.pointcloud2_cdr is the fixed
    x, y, z, intensity layout of the node cloud; cdr_oracle.parse_pointcloud2 reads any field list.)"""
    raw = bytes(np.ascontiguousarray(data).view(np.uint8).reshape(-1))
    assert len(raw) == width * point_step
    w = CDR._W()
    w.header(sec, nanosec, frame_id)
    w.prim("I", 1)      # height
    w.prim("I", width)
    w.prim("I", len(fields))
    for name, offset, datatype, count in fields:
        w.string(name)
        w.prim("I", offset)
        w.prim("B", datatype)
        w.prim("I", count)
    w.prim("B", 0)      # is_bigendian
    w.prim("I", point_step)
    w.prim("I", point_step * width)  # row_step
    w.prim("I", len(raw))
    w.b += raw
    w.prim("B", is_dense)
    return bytes(w.b)


def cloud_records(msg: dict) -> np.ndarray:
    """The points of a parsed PointCloud2 (cdr_oracle.parse_pointcloud2) as a structured array of its fields (count 1
    each)."""
    dt = np.dtype({"names": [f[0] for f in msg["fields"]], "formats": [_FIELD_FMT[f[2]] for f in msg["fields"]],
                   "offsets": [f[1] for f in msg["fields"]], "itemsize": msg["point_step"]})
    assert all(f[3] == 1 for f in msg["fields"]) and msg["height"] == 1
    return np.frombuffer(msg["data"].tobytes(), dt, msg["width"])


def params(channels=DEFAULT, range_cutoff=-1.0):
    """the attributes of rpl_scan_cloud_params (range_cutoff as the float32 the struct holds)"""
    return SimpleNamespace(channels=int(channels), range_cutoff=float(np.float32(range_cutoff)))


def params_ok(p) -> bool:
    """the rules rpl_scan_cloud_batch_dev and rpl_capsule_stream_scan_cloud_msgs enforce"""
    return (int(p.channels) & ~CHANNELS) == 0 and not np.isnan(np.float32(p.range_cutoff))


def fields(channels):
    """[(name, offset, datatype, count)] of a channel set"""
    names = [("x", FLOAT32), ("y", FLOAT32), ("z", FLOAT32)]
    names += [(n, t) for bit, n, t in CHANNEL_FIELDS if channels & bit]
    return [(n, 4 * k, t, 1) for k, (n, t) in enumerate(names)]


def point_step(channels) -> int:
    return 12 + 4 * bin(int(channels) & CHANNELS).count("1")


def cutoff(p, range_max) -> np.float32:
    return np.float32(p.range_cutoff) if np.float32(p.range_cutoff) >= 0 else np.float32(range_max)


def kept(p, ranges, range_min, range_max):
    """the kept beams' mask"""
    r = np.asarray(ranges, np.float32)
    with np.errstate(invalid="ignore"):
        return (r >= np.float32(range_min)) & (r < cutoff(p, range_max))


def project(p, ranges, intensities, inc, time_increment, range_min, range_max) -> np.ndarray:
    """the records of P: [width, point_step] uint8 (little endian words)"""
    assert params_ok(p)
    r = np.asarray(ranges, np.float32)
    keep = kept(p, r, range_min, range_max)
    idx = np.nonzero(keep)[0]
    x, y = SFP.beam_points(np.where(keep, r, np.float32(0)), inc)
    cols = [x[idx].view(np.uint32), y[idx].view(np.uint32), np.zeros(idx.shape[0], np.uint32)]
    if p.channels & INTENSITY:
        cols.append(np.asarray(intensities, np.float32)[idx].view(np.uint32))
    if p.channels & INDEX:
        cols.append(idx.astype(np.int32).view(np.uint32))
    if p.channels & DISTANCE:
        cols.append(r[idx].view(np.uint32))
    if p.channels & TIMESTAMP:
        cols.append((idx.astype(np.float32) * np.float32(time_increment)).astype(np.float32).view(np.uint32))
    words = np.stack(cols, axis=1).astype("<u4") if idx.shape[0] else np.zeros((0, len(cols)), "<u4")
    return words.view(np.uint8).reshape(idx.shape[0], point_step(p.channels))


def P(p, scan: dict) -> bytes:
    """the PointCloud2 message of one LaserScan message (scan: cdr_oracle.parse_laserscan's dict)"""
    assert float(scan["angle_min"]) == 0.0
    rec = project(p, scan["ranges"], scan["intensities"], scan["angle_increment"], scan["time_increment"],
                  scan["range_min"], scan["range_max"])
    return pointcloud2_fields_cdr(scan["sec"], scan["nanosec"], scan["frame_id"], fields(p.channels),
                                  point_step(p.channels), rec, rec.shape[0])


def project_rows(p, ranges, intensities, beam_counts, angle_increment, time_increment, range_min, range_max):
    """P over padded rows [n, stride] (rpl_scan_cloud_batch_dev): ([records per row], kept counts); time_increment
    None: 0"""
    out, counts = [], []
    for s in range(ranges.shape[0]):
        M = int(beam_counts[s])
        ti = 0.0 if time_increment is None else time_increment[s]
        rec = project(p, ranges[s, :M], intensities[s, :M], angle_increment[s], ti, range_min, range_max)
        out.append(rec)
        counts.append(rec.shape[0])
    return out, np.asarray(counts, np.uint32)
