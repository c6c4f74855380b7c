"""The LaserScan filter chain F(settings, scan), restated on the CPU in numpy float32 (DESIGN.md 5.7.1 "LaserScan
filters").  This docstring is the definition; csrc/scan_filter.cu computes the same bits.

F maps one published LaserScan -- ranges[0..M), intensities[0..M), angle_increment inc, angle_min 0, Mode A or B and
the inversion already applied -- to a LaserScan of the same beam count and increment.  A removed beam's range becomes
the quiet NaN 0x7FC00000 (REP 117: erroneous detection); its intensity is unchanged.  A beam whose range is already
non-finite (Mode A's +inf empty bins, an earlier stage's NaN) is never tested and never changed.

The stages run in this order; each reads the whole output of the one before and decides every beam from it alone:
  1. angular mask: beam i is removed when a_i = fl(float(i) * inc) lies in a sector, lo_k <= a_i <= hi_k, of the four
     [mask_lo[k], mask_hi[k]] (radians in the published frame; lo > hi: unused; a sector through 0 is two sectors);
  2. range window: a finite r_i < range_lo or r_i > range_hi is removed;
  3. intensity floor: intensity_i < intensity_min is removed (the cloud chain's keep intensity >= intensity_min);
  4. speckle: a finite r_i is kept iff at least speckle_min_neighbours beams j, 1 <= |j - i| <= speckle_window,
     0 <= j < M, have a finite r_j with |fl(r_j - r_i)| <= speckle_max_diff (no wrap from beam M-1 to beam 0);
  5. veiling points: for beams i, j with 1 <= |j - i| = k <= shadow_window, both finite and > 0, and r_i < r_j, the far
     beam j is removed when dx = fl(fl(r_j * c_k) - r_i) > 0 and fl(r_j * s_k) < fl(tan_shadow * dx): the segment from
     p_i = (r_i, 0) to p_j = (r_j c_k, r_j s_k) makes an angle below shadow_angle with the line of sight through p_i.
Every float operation is rounded as written (no FMA).  tan_shadow = float(tan(double(shadow_angle))), computed once on
the host.  (s_k, c_k) = float(sincos(double(k) * double(inc))) by sincos_f64 below: Cody-Waite reduction by pi/2 and
fdlibm's kernel polynomials, every double operation rounded as written, in the kernel and here alike.

A stage with window 0 is off.  Limits: windows <= 16, speckle_min_neighbours <= 2 * speckle_window, shadow_angle in
(0, pi/2) when the shadow stage is on, range_lo <= range_hi, no NaN anywhere; settings_ok tells.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

NAN_BITS = 0x7FC00000
MAX_WINDOW = 16
MAX_BEAMS = 8192

# Cody-Waite split of pi/2: the first 33 bits (k * PIO2_1 is exact for |k| < 2^20) and the rest; fdlibm's pio2_1, pio2_1t
TWO_OVER_PI = 6.36619772367581382433e-01
PIO2_1 = 1.57079632673412561417e+00
PIO2_1T = 6.07710050650619224932e-11
# fdlibm __kernel_sin / __kernel_cos coefficients on [-pi/4, pi/4]
S = (-1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04,
     2.75573137070700676789e-06, -2.50507602534068634195e-08, 1.58969099521155010221e-10)
C = (4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05,
     -2.75573143513906633035e-07, 2.08757232129817482790e-09, -1.13596475577881948265e-11)


def settings(mask=(), range_lo=-math.inf, range_hi=math.inf, intensity_min=-math.inf, speckle_window=0,
             speckle_min_neighbours=0, speckle_max_diff=0.0, shadow_window=0, shadow_angle=0.0, enabled=True):
    """An entry with the attributes of rpl_scan_filter_settings; mask: up to four (lo, hi) sectors."""
    assert len(mask) <= 4
    lo = [float(a) for a, _ in mask] + [math.inf] * (4 - len(mask))
    hi = [float(b) for _, b in mask] + [-math.inf] * (4 - len(mask))
    return SimpleNamespace(mask_lo=lo, mask_hi=hi, range_lo=float(range_lo), range_hi=float(range_hi),
                           intensity_min=float(intensity_min), speckle_max_diff=float(speckle_max_diff),
                           shadow_angle=float(shadow_angle), speckle_window=int(speckle_window),
                           speckle_min_neighbours=int(speckle_min_neighbours), shadow_window=int(shadow_window),
                           enabled=int(bool(enabled)))


def _f32(x):
    return np.float32(x)


def settings_ok(s) -> bool:
    """The limits rpl_scan_filter_batch_dev and rpl_capsule_stream_set_scan_filters enforce."""
    floats = [_f32(v) for v in list(s.mask_lo) + list(s.mask_hi)] + [
        _f32(s.range_lo), _f32(s.range_hi), _f32(s.intensity_min), _f32(s.speckle_max_diff), _f32(s.shadow_angle)]
    if any(np.isnan(v) for v in floats):
        return False
    if s.speckle_window > MAX_WINDOW or s.shadow_window > MAX_WINDOW:
        return False
    if s.speckle_min_neighbours > 2 * s.speckle_window:
        return False
    if not _f32(s.range_lo) <= _f32(s.range_hi):
        return False
    if s.shadow_window > 0 and not (0.0 < float(_f32(s.shadow_angle)) < math.pi / 2):
        return False
    return True


def tan_shadow(s) -> np.float32:
    return _f32(math.tan(float(_f32(s.shadow_angle))))


def sincos_f64(x):
    """(sin x, cos x) in double, every operation rounded as written; x >= 0, x < 2^20 * pi / 2 (scalar or array)."""
    x = np.asarray(x, dtype=np.float64)
    q = np.rint(x * TWO_OVER_PI)
    r = (x - q * PIO2_1) - q * PIO2_1T
    z = r * r
    ps = S[0] + z * (S[1] + z * (S[2] + z * (S[3] + z * (S[4] + z * S[5]))))
    pc = C[0] + z * (C[1] + z * (C[2] + z * (C[3] + z * (C[4] + z * C[5]))))
    sn = r + (r * z) * ps
    cs = (1.0 - 0.5 * z) + (z * z) * pc
    n = q.astype(np.int64) & 3
    sin = np.select([n == 0, n == 1, n == 2], [sn, cs, -sn], -cs)
    cos = np.select([n == 0, n == 1, n == 2], [cs, -sn, -cs], sn)
    return sin, cos


def sincos_table(inc, window):
    """float32 (s_k, c_k) for k = 0..window (entry 0 unused)"""
    k = np.arange(window + 1, dtype=np.float64)
    s, c = sincos_f64(k * float(np.float32(inc)))
    s, c = s.astype(np.float32), c.astype(np.float32)
    s[0] = c[0] = 0
    return s, c


def _nan():
    return np.array([NAN_BITS], np.uint32).view(np.float32)[0]


def _neighbour(r, d):
    """(r[i + d], whether 0 <= i + d < M) for every i"""
    M = r.shape[0]
    j = np.arange(M) + d
    ok = (j >= 0) & (j < M)
    return r[np.clip(j, 0, M - 1)], ok


def removed_pointwise(s, r, it, inc):
    """stages 1-3 on ranges r: the beams they remove"""
    M = r.shape[0]
    a = np.arange(M).astype(np.float32) * np.float32(inc)
    rm = np.zeros(M, bool)
    for lo, hi in zip(s.mask_lo, s.mask_hi):
        rm |= (_f32(lo) <= a) & (a <= _f32(hi))
    rm |= (r < _f32(s.range_lo)) | (r > _f32(s.range_hi))
    rm |= np.asarray(it, np.float32) < _f32(s.intensity_min)
    return rm & np.isfinite(r)


def removed_speckle(s, r):
    """stage 4 on ranges r: the beams it removes"""
    W = int(s.speckle_window)
    cnt = np.zeros(r.shape[0], np.int64)
    D = _f32(s.speckle_max_diff)
    for d in [e for e in range(-W, W + 1) if e != 0]:
        rj, ok = _neighbour(r, d)
        with np.errstate(invalid="ignore", over="ignore"):
            cnt += (ok & np.isfinite(rj) & (np.abs(rj - r) <= D)).astype(np.int64)
    return np.isfinite(r) & (cnt < int(s.speckle_min_neighbours))


def removed_veiling(s, r, inc):
    """stage 5 on ranges r: the far beams j it removes"""
    K = int(s.shadow_window)
    sk, ck = sincos_table(inc, K)
    t = tan_shadow(s)
    pos = np.isfinite(r) & (r > 0)
    rm = np.zeros(r.shape[0], bool)
    for k in range(1, K + 1):
        for d in (-k, k):
            ri, ok = _neighbour(r, d)
            pi, _ = _neighbour(pos, d)
            with np.errstate(invalid="ignore", over="ignore"):
                dx = r * ck[k] - ri
                rm |= ok & pos & pi & (ri < r) & (dx > 0) & (r * sk[k] < t * dx)
    return rm


def filter_scan(s, ranges, intensities, inc):
    """F(s, scan): the filtered ranges (float32, same length); intensities are not changed.  A disabled entry returns
    the ranges as they are."""
    r = np.array(ranges, dtype=np.float32, copy=True)
    if not s.enabled or r.shape[0] == 0:
        return r
    with np.errstate(invalid="ignore", over="ignore"):
        r[removed_pointwise(s, r, intensities, inc)] = _nan()
        if s.speckle_window > 0:
            r[removed_speckle(s, r)] = _nan()
        if s.shadow_window > 0:
            r[removed_veiling(s, r, inc)] = _nan()
    return r


def filter_rows(entries, ranges, intensities, beam_counts, angle_increment, per=None):
    """F over padded rows [n, stride]: row s takes entries[s // per] (per None: one entry for every row).  Returns the
    filtered copy of ranges."""
    out = np.array(ranges, dtype=np.float32, copy=True)
    for s in range(out.shape[0]):
        e = entries if per is None else entries[s // per]
        M = int(beam_counts[s])
        if M:
            out[s, :M] = filter_scan(e, out[s, :M], intensities[s, :M], angle_increment[s])
    return out
