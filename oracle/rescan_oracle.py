"""LaserScans re-gridded from the projected clouds (DESIGN.md 5.7.1 "LaserScans re-gridded from the projected clouds"),
pointcloud_to_laserscan's PointCloudToLaserScanNode::cloudCallback, restated on the CPU in numpy.  This docstring is the
definition; csrc/rescan.cu computes the same bits.

Q(settings, cloud) is a pure function of one PointCloud2's x, y, z.  In a session the cloud is slot i's message of
scan_cloud_msgs with the same scan and cloud params: Q is composed onto P (oracle/scan_cloud_oracle.py) and onto the
transform rule of tests/scan_cloud_transform_oracle.py, and the points it tests are exactly the records those publish.

  grid:  ranges_size = ceil(fl32(fl32(angle_max - angle_min) / angle_increment)): the message's float fields, as the
         package computes it.
  seed:  every beam starts at +inf when use_inf is set, else at fl32(range_max + inf_epsilon) (the sum in double, as
         the package adds its double inf_epsilon to the message's float range_max).
  point: each (X, Y, Z), in record order:
         1. skipped when Z > max_height or Z < min_height;
         2. range = sqrt(fl64(X*X + Y*Y)) in double: the products are exact for float inputs, the sum is rounded once
            and sqrt is correctly rounded (reproducible on both sides, unlike libm's hypot);
         3. skipped when range < range_min or range > range_max;
         4. angle = atan2_f64(Y, X), skipped when angle < angle_min or angle > angle_max;
         5. index = (int) fl64(fl64(angle - angle_min) / angle_increment), skipped when index >= ranges_size (the
            package would write past its grid there);
         6. ranges[index] = fl32(range) when range < ranges[index].  Rounding is monotonic, so the float min is the
            double min rounded, and the order of the points does not matter.
  atan2_f64: fdlibm's atan and atan2 (the atanhi / atanlo tables, the 11 aT coefficients, the quadrant and signed-zero
         cases), every double operation rounded as written, no FMA; the family of sincos_f64 in
         oracle/scan_filter_oracle.py.  The device's copy sits next to sincos_f64 in csrc/beam_point.cuh.
  message: sensor_msgs/LaserScan with the cloud's stamp and frame_id (the stream's target frame under an enabled
         transform entry, else the LaserScan's); angle_min, angle_max, angle_increment, scan_time, range_min,
         range_max the entry's; time_increment 0; ranges_size ranges; no intensities (the package publishes none).  A
         cloud of width 0 gives every beam its seed.  A disabled entry gives no message.
  limits: every float finite, angle_increment > 0, angle_min < angle_max, 1 <= ranges_size <= 8192 (a slot's grid
         fits in shared memory), 0 <= range_min <= range_max, min_height <= max_height, inf_epsilon >= 0; anything
         else is refused (RPL_RESULT_INVALID_DATA).

The package's loop is restated from memory of its source, which was not at hand when this was written (as the field
names of oracle/scan_cloud_oracle.py): these bytes are the definition either way.  target_frame comes through the
transform table; transform_tolerance and queue_size have no meaning on the device; concurrency_level is not served.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

from oracle import cdr_oracle as CDR

MAX_BINS = 8192
FLT_MAX = float(np.finfo(np.float32).max)

# fdlibm s_atan.c
ATANHI = (4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01,
          1.57079632679489655800e+00)
ATANLO = (2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17,
          6.12323399573676603587e-17)
AT = (3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01,
      -1.11111104054623557880e-01, 9.09088713343650656196e-02, -7.69187620504482999495e-02,
      6.66107313738753120669e-02, -5.83357013379057348645e-02, 4.97687799461593236017e-02,
      -3.65315727442169155270e-02, 1.62858201153657823623e-02)
# fdlibm e_atan2.c
TINY, PI_O_4, PI_O_2, PI, PI_LO = 1.0e-300, 7.8539816339744827900e-01, 1.5707963267948965580e+00, \
    3.1415926535897931160e+00, 1.2246467991473531772e-16


def settings(angle_min=-math.pi, angle_max=math.pi, angle_increment=math.pi / 180.0, range_min=0.0, range_max=FLT_MAX,
             min_height=-FLT_MAX, max_height=FLT_MAX, use_inf=True, inf_epsilon=1.0, scan_time=1.0 / 30.0,
             enabled=True):
    """the attributes of rpl_rescan_settings, each float as the float32 the struct holds"""
    f = lambda v: float(np.float32(v))  # noqa: E731
    return SimpleNamespace(angle_min=f(angle_min), angle_max=f(angle_max), angle_increment=f(angle_increment),
                           range_min=f(range_min), range_max=f(range_max), min_height=f(min_height),
                           max_height=f(max_height), inf_epsilon=f(inf_epsilon), scan_time=f(scan_time),
                           use_inf=bool(use_inf), enabled=bool(enabled))


def ranges_size(s) -> int:
    """ceil(fl32(fl32(angle_max - angle_min) / angle_increment)); 0 when that is not a count in [1, MAX_BINS]"""
    f = np.float32
    with np.errstate(all="ignore"):
        q = np.ceil(f(f(f(s.angle_max) - f(s.angle_min)) / f(s.angle_increment)))
    return int(q) if 1 <= q <= MAX_BINS else 0


def settings_ok(s) -> bool:
    """the limits rpl_rescan_batch_dev and rpl_capsule_stream_set_rescans enforce (on an enabled entry)"""
    v = [s.angle_min, s.angle_max, s.angle_increment, s.range_min, s.range_max, s.min_height, s.max_height,
         s.inf_epsilon, s.scan_time]
    if not all(math.isfinite(x) for x in v):
        return False
    if not (s.angle_increment > 0 and s.angle_min < s.angle_max) or ranges_size(s) == 0:
        return False
    return 0 <= s.range_min <= s.range_max and s.min_height <= s.max_height and s.inf_epsilon >= 0


def seed(s) -> np.float32:
    return np.float32(np.inf) if s.use_inf else np.float32(float(s.range_max) + float(s.inf_epsilon))


def _words(x):
    """(high word as int32, low word as uint32) of each double"""
    u = np.asarray(x, np.float64).view(np.uint64)
    return (u >> np.uint64(32)).astype(np.uint32).view(np.int32).astype(np.int64), (u & np.uint64(0xFFFFFFFF)).astype(
        np.int64)


def atan_f64(x):
    """fdlibm's atan, every operation rounded as written (array or scalar)"""
    x = np.asarray(x, np.float64)
    hx, _ = _words(x)
    ix = hx & 0x7FFFFFFF
    a = np.abs(x)
    with np.errstate(all="ignore"):
        ids = np.select([ix < 0x3FDC0000, ix < 0x3FE60000, ix < 0x3FF30000, ix < 0x40038000], [-1, 0, 1, 2], 3)
        xr = np.select([ids == -1, ids == 0, ids == 1, ids == 2],
                       [x, (2.0 * a - 1.0) / (2.0 + a), (a - 1.0) / (a + 1.0), (a - 1.5) / (1.0 + 1.5 * a)], -1.0 / a)
        z = xr * xr
        w = z * z
        s1 = z * (AT[0] + w * (AT[2] + w * (AT[4] + w * (AT[6] + w * (AT[8] + w * AT[10])))))
        s2 = w * (AT[1] + w * (AT[3] + w * (AT[5] + w * (AT[7] + w * AT[9]))))
        xs = xr * (s1 + s2)
        k = np.clip(ids, 0, 3)
        r = np.asarray(ATANHI)[k] - ((xs - np.asarray(ATANLO)[k]) - xr)
        out = np.where(ids < 0, xr - xs, np.where(hx < 0, -r, r))
        out = np.where(ix < 0x3E200000, x, out)
        big = np.where(hx > 0, ATANHI[3] + ATANLO[3], -ATANHI[3] - ATANLO[3])
        out = np.where(ix >= 0x44100000, np.where(np.isnan(x), x + x, big), out)
    return out[()] if out.ndim == 0 else out


def atan2_f64(y, x):
    """fdlibm's atan2 (__ieee754_atan2), every operation rounded as written (arrays or scalars, broadcast)"""
    y, x = np.broadcast_arrays(np.asarray(y, np.float64), np.asarray(x, np.float64))
    hx, lx = _words(x)
    hy, ly = _words(y)
    ix, iy = hx & 0x7FFFFFFF, hy & 0x7FFFFFFF
    m = (np.signbit(y).astype(np.int64)) | (np.signbit(x).astype(np.int64) << 1)
    k = (iy - ix) >> 20
    with np.errstate(all="ignore"):
        z = atan_f64(np.abs(y / x))
        z = np.where(k > 60, PI_O_2 + 0.5 * PI_LO, np.where((hx < 0) & (k < -60), 0.0, z))
        general = np.select([m == 0, m == 1, m == 2], [z, -z, PI - (z - PI_LO)], (z - PI_LO) - PI)
        y_zero = np.select([m < 2, m == 2], [y, np.full_like(y, PI + TINY)], -PI - TINY)
        half = np.where(hy < 0, -PI_O_2 - TINY, PI_O_2 + TINY)
        both_inf = np.select([m == 0, m == 1, m == 2], [PI_O_4 + TINY, -PI_O_4 - TINY, 3.0 * PI_O_4 + TINY],
                             -3.0 * PI_O_4 - TINY)
        x_inf = np.select([m == 0, m == 1, m == 2], [0.0, -0.0, PI + TINY], -PI - TINY)
        out = np.select(
            [np.isnan(x) | np.isnan(y), x == 1.0, y == 0.0, x == 0.0, np.isinf(x) & np.isinf(y), np.isinf(x),
             np.isinf(y)],
            [x + y, atan_f64(y), y_zero, half, both_inf, x_inf, half], general)
    return out[()] if out.ndim == 0 else out


def range_f64(x, y):
    """sqrt(fl64(X*X + Y*Y)) of float32 coordinates"""
    X, Y = np.asarray(x, np.float32).astype(np.float64), np.asarray(y, np.float32).astype(np.float64)
    return np.sqrt(X * X + Y * Y)


def regrid(s, x, y, z) -> np.ndarray:
    """the ranges of Q for the points (x, y, z) (float32 arrays in record order): float32 [ranges_size]"""
    n = ranges_size(s)
    assert settings_ok(s)
    out = np.full(n, seed(s), np.float32)
    x, y, z = (np.asarray(v, np.float32).reshape(-1) for v in (x, y, z))
    keep = ~((z > np.float32(s.max_height)) | (z < np.float32(s.min_height)))
    r = range_f64(x, y)
    keep &= ~((r < s.range_min) | (r > s.range_max))
    a = atan2_f64(y.astype(np.float64), x.astype(np.float64))
    with np.errstate(invalid="ignore"):
        keep &= ~((a < s.angle_min) | (a > s.angle_max))
        q = (a - s.angle_min) / s.angle_increment
    idx = np.where(keep, q, 0.0).astype(np.int64)  # truncation toward zero; q >= 0 where kept
    keep &= idx < n
    np.minimum.at(out, idx[keep], r[keep].astype(np.float32))
    return out


def cloud_xyz(msg: dict):
    """x, y, z of a parsed PointCloud2 (cdr_oracle.parse_pointcloud2) whose first three fields are x, y, z"""
    assert [f[0] for f in msg["fields"][:3]] == ["x", "y", "z"]
    w = msg["data"].view("<f4").reshape(msg["width"], msg["point_step"] // 4) if msg["width"] else \
        np.zeros((0, 3), "<f4")
    return w[:, 0], w[:, 1], w[:, 2]


def Q(s, cloud: dict):
    """the LaserScan message (bytes) of one parsed PointCloud2 under entry s; None for a disabled entry"""
    if not s.enabled:
        return None
    ranges = regrid(s, *cloud_xyz(cloud))
    scal = (s.angle_min, s.angle_max, s.angle_increment, 0.0, s.scan_time, s.range_min, s.range_max)
    return CDR.laserscan_cdr(cloud["sec"], cloud["nanosec"], cloud["frame_id"], scal, ranges,
                             np.zeros(0, np.float32))
