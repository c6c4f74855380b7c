"""CPU checks of the LaserScan filter chain's definition (oracle/scan_filter_oracle.py): hand-built scans for every
stage, the float32 restatement against an independent float64 statement of each stage, and the (sin, cos) polynomial
against numpy over every angle the veiling stage can meet."""
import math

import numpy as np
import pytest

from oracle import scan_filter_oracle as F

INC360 = np.float32(2 * math.pi / 360)


def _removed(out):
    return np.flatnonzero(np.isnan(out))


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_veiling_streak_behind_an_edge():
    # background at 5 m, an object at 2 m over beams 40..59, mixed pixels 60..63 between it and the background
    r = np.full(360, 5.0, np.float32)
    r[40:60] = 2.0
    r[60:64] = [2.03, 2.3, 2.6, 3.0]
    it = np.full(360, 10.0, np.float32)
    s = F.settings(shadow_window=4, shadow_angle=math.radians(10))
    out = F.filter_scan(s, r, it, INC360)
    rm = set(_removed(out).tolist())
    # the object itself stays, the streak's far beams go
    assert not rm & set(range(40, 60))
    assert {61, 62, 63} <= rm
    # 2.03 m one beam behind 2 m: dx = 2.03 cos(1 deg) - 2 = 0.0297, dy = 0.0354: 50 degrees, kept
    assert 60 not in rm
    # the background beyond the streak's first beam, and in front of the object's left edge, as defined: the far beam of
    # every depth jump within the window whose segment is nearly along the line of sight
    for j in list(range(36, 40)) + list(range(64, 68)):
        near = [i for i in range(j - 4, j + 5) if i != j and r[i] < r[j]]
        expect = False
        for i in near:
            k = abs(i - j)
            dx = r[j] * math.cos(k * INC360) - r[i]
            expect |= dx > 0 and math.atan2(r[j] * math.sin(k * INC360), dx) < math.radians(10)
        assert (j in rm) == expect, j
    assert not rm & set(range(70, 360))
    assert (_bits(out[60]) == _bits(r[60])).all()
    assert (_bits(out[list(rm)]) == F.NAN_BITS).all()


def test_single_speckle_removed_and_two_beam_cluster_kept():
    r = np.full(200, 5.0, np.float32)
    r[50] = 1.0           # a speckle
    r[120:122] = [1.0, 1.02]  # a two-beam cluster
    it = np.ones(200, np.float32)
    s = F.settings(speckle_window=2, speckle_min_neighbours=1, speckle_max_diff=0.05)
    out = F.filter_scan(s, r, it, INC360)
    assert _removed(out).tolist() == [50]
    # two neighbours needed: the cluster goes too, the background stays
    s2 = F.settings(speckle_window=2, speckle_min_neighbours=2, speckle_max_diff=0.05)
    assert _removed(F.filter_scan(s2, r, it, INC360)).tolist() == [50, 120, 121]


def test_masked_sectors():
    r = np.full(360, 3.0, np.float32)
    it = np.ones(360, np.float32)
    a = np.arange(360, dtype=np.float32) * INC360
    s = F.settings(mask=[(0.5, 1.0)])
    assert (np.isnan(F.filter_scan(s, r, it, INC360)) == ((a >= np.float32(0.5)) & (a <= np.float32(1.0)))).all()
    # a sector through 0, given as two sectors: [-0.2, 0.2] as [0, 0.2] and [2 pi - 0.2, 2 pi]
    s = F.settings(mask=[(0.0, 0.2), (2 * math.pi - 0.2, 2 * math.pi)])
    got = np.isnan(F.filter_scan(s, r, it, INC360))
    want = (a <= np.float32(0.2)) | (a >= np.float32(2 * math.pi - 0.2))
    assert (got == want).all() and got[0] and got[359] and not got[180]
    # lo > hi: an unused sector
    assert not np.isnan(F.filter_scan(F.settings(mask=[(1.0, 0.5)]), r, it, INC360)).any()


def test_range_window_and_intensity_floor():
    r = np.array([0.1, 0.15, 1.0, 12.0, 12.5, 3.0], np.float32)
    it = np.array([5, 5, 5, 5, 5, 0.5], np.float32)
    s = F.settings(range_lo=0.15, range_hi=12.0, intensity_min=1.0)
    assert _removed(F.filter_scan(s, r, it, INC360)).tolist() == [0, 4, 5]


def test_non_finite_inputs_pass_untouched():
    r = np.full(64, 2.0, np.float32)
    odd_nan = np.array([0x7FC00123], np.uint32).view(np.float32)[0]
    r[[3, 4, 5]] = [np.inf, odd_nan, -np.inf]
    r[10] = 30.0
    it = np.zeros(64, np.float32)
    s = F.settings(mask=[(0.0, 1.0)], range_lo=0.5, range_hi=10.0, intensity_min=1.0, speckle_window=3,
                   speckle_min_neighbours=6, speckle_max_diff=0.1, shadow_window=16, shadow_angle=0.5)
    out = F.filter_scan(s, r, it, INC360)
    assert (_bits(out[[3, 4, 5]]) == _bits(r[[3, 4, 5]])).all()
    assert (_bits(np.delete(out, [3, 4, 5])) == F.NAN_BITS).all()
    # disabled: nothing changes
    s.enabled = 0
    assert (_bits(F.filter_scan(s, r, it, INC360)) == _bits(r)).all()


@pytest.mark.parametrize("M", [1, 2, 3])
def test_tiny_scans(M):
    r = np.array([1.0, 3.0, 1.01][:M], np.float32)
    it = np.ones(M, np.float32)
    inc = np.float32(2 * math.pi / max(M - 1, 1))
    keep_all = F.settings(speckle_window=1, speckle_min_neighbours=0, speckle_max_diff=0.1)
    assert (_bits(F.filter_scan(keep_all, r, it, inc)) == _bits(r)).all()
    s = F.settings(speckle_window=2, speckle_min_neighbours=1, speckle_max_diff=0.1)
    out = F.filter_scan(s, r, it, inc)
    assert out.shape == (M,)
    assert _removed(out).tolist() == {1: [0], 2: [0, 1], 3: [1]}[M]  # beams 0 and 2 are 2 apart: window 2 pairs them
    v = F.filter_scan(F.settings(shadow_window=16, shadow_angle=1.5), r, it, inc)
    assert v.shape == (M,)


# ---- the restatement against an independent float64 statement, stage by stage on the same input --------------------
def _f64_pointwise(s, r, it, inc):
    a = np.arange(len(r)) * float(inc)
    rm, margin = np.zeros(len(r), bool), np.full(len(r), np.inf)
    for lo, hi in zip(s.mask_lo, s.mask_hi):
        rm |= (lo <= a) & (a <= hi)
        with np.errstate(invalid="ignore"):
            margin = np.minimum(margin, np.minimum(np.abs(a - lo), np.abs(a - hi)) / np.maximum(np.abs(a), 1e-30))
    rm |= (r < s.range_lo) | (r > s.range_hi) | (it < s.intensity_min)
    return rm & np.isfinite(r), np.nan_to_num(margin, nan=np.inf)


def _f64_speckle(s, r):
    M, W = len(r), s.speckle_window
    rm, margin = np.zeros(M, bool), np.full(M, np.inf)
    for i in range(M):
        if not np.isfinite(r[i]):
            continue
        cnt = 0
        for j in range(max(0, i - W), min(M, i + W + 1)):
            if j != i and np.isfinite(r[j]):
                d = abs(float(r[j]) - float(r[i]))
                cnt += d <= s.speckle_max_diff
                margin[i] = min(margin[i], abs(d - s.speckle_max_diff) / max(s.speckle_max_diff, 1e-30))
        rm[i] = cnt < s.speckle_min_neighbours
    return rm, margin


def _f64_veiling(s, r, inc):
    M, K = len(r), s.shadow_window
    rm, margin = np.zeros(M, bool), np.full(M, np.inf)
    t = math.tan(s.shadow_angle)
    for j in range(M):
        rj = float(r[j])
        if not (np.isfinite(rj) and rj > 0):
            continue
        for i in range(max(0, j - K), min(M, j + K + 1)):
            ri = float(r[i])
            if i == j or not (np.isfinite(ri) and 0 < ri < rj):
                continue
            k = abs(i - j)
            dx = rj * math.cos(k * float(inc)) - ri
            dy = rj * math.sin(k * float(inc))
            rm[j] |= dx > 0 and dy < t * dx
            margin[j] = min(margin[j], abs(dx) / rj, abs(dy - t * dx) / rj)
    return rm, margin


def _random_scan(rng, M):
    r = rng.uniform(0.1, 12.0, M).astype(np.float32)
    # walls: runs of slowly changing range, with jumps between them
    walls = np.cumsum(rng.random(M) < 0.05)
    base = rng.uniform(0.5, 10.0, walls.max() + 1).astype(np.float32)
    r = np.where(rng.random(M) < 0.9, base[walls] + rng.normal(0, 0.01, M).astype(np.float32), r).astype(np.float32)
    r[rng.random(M) < 0.05] = np.inf
    it = rng.uniform(0, 60, M).astype(np.float32)
    return r, it


def _random_settings(rng):
    sectors = []
    for _ in range(int(rng.integers(0, 5))):
        lo = float(rng.uniform(0, 2 * math.pi))
        sectors.append((lo, lo + float(rng.uniform(-0.5, 1.0))))
    lo = float(rng.uniform(0, 1.0))
    return F.settings(mask=sectors, range_lo=lo, range_hi=lo + float(rng.uniform(0, 12)),
                      intensity_min=float(rng.uniform(0, 20)), speckle_window=(w := int(rng.integers(0, 17))),
                      speckle_min_neighbours=int(rng.integers(0, 2 * w + 1)), speckle_max_diff=float(rng.uniform(0, 0.3)),
                      shadow_window=int(rng.integers(0, 17)), shadow_angle=float(rng.uniform(0.01, 1.5)))


@pytest.mark.parametrize("seed", range(8))
def test_restatement_against_float64(seed):
    rng = np.random.default_rng(seed)
    near, total = 0, 0
    for _ in range(3):
        M = int(rng.integers(2, 2000))
        inc = np.float32(2 * math.pi / (M if rng.random() < 0.5 else M - 1))
        r, it = _random_scan(rng, M)
        s = _random_settings(rng)
        assert F.settings_ok(s)
        got = F.removed_pointwise(s, r, it, inc)
        want, margin = _f64_pointwise(s, r, it, inc)
        bad = got != want
        assert (margin[bad] < 1e-6).all()
        near += int(bad.sum())
        r = r.copy()
        r[got] = np.nan
        if s.speckle_window:
            got = F.removed_speckle(s, r)
            want, margin = _f64_speckle(s, r)
            bad = got != want
            assert (margin[bad] < 1e-6).all()
            near += int(bad.sum())
            r[got] = np.nan
        s.shadow_window = max(s.shadow_window, 1)
        with np.errstate(invalid="ignore"):
            got = F.removed_veiling(s, r, inc)
        want, margin = _f64_veiling(s, r, inc)
        bad = got != want
        assert (margin[bad] < 1e-6).all()
        near += int(bad.sum())
        total += 3 * M
    assert near <= max(2, total // 1000)


def test_sincos_polynomial_within_one_ulp():
    M = np.arange(2, 8193, dtype=np.float64)
    incs = np.concatenate([(2 * np.pi / M).astype(np.float32), (2 * np.pi / (M - 1)).astype(np.float32)])
    k = np.arange(1, 17, dtype=np.float64)
    x = (k[None, :] * incs.astype(np.float64)[:, None]).ravel()
    s, c = F.sincos_f64(x)
    for got, ref in ((s, np.sin(x)), (c, np.cos(x))):
        g, e = got.astype(np.float32), ref.astype(np.float32)
        ulps = np.abs(g.view(np.int32).astype(np.int64) - e.view(np.int32).astype(np.int64))
        # (a sign change at a zero crossing is no ulp distance: compare those by value)
        same_sign = np.signbit(g) == np.signbit(e)
        assert (ulps[same_sign] <= 1).all()
        assert (np.abs(g - e)[~same_sign] <= np.spacing(np.float32(1e-30))).all() if (~same_sign).any() else True


def test_settings_limits():
    ok = F.settings(speckle_window=16, speckle_min_neighbours=32, shadow_window=16, shadow_angle=1.5, range_lo=1,
                    range_hi=1)
    assert F.settings_ok(ok)
    assert F.settings_ok(F.settings())
    bad = [
        F.settings(speckle_window=17),
        F.settings(shadow_window=17, shadow_angle=0.5),
        F.settings(speckle_window=2, speckle_min_neighbours=5),
        F.settings(shadow_window=1, shadow_angle=0.0),
        F.settings(shadow_window=1, shadow_angle=math.pi / 2),
        F.settings(shadow_window=1, shadow_angle=-0.1),
        F.settings(range_lo=2.0, range_hi=1.0),
        F.settings(range_lo=math.nan),
        F.settings(intensity_min=math.nan),
        F.settings(speckle_max_diff=math.nan),
        F.settings(mask=[(math.nan, 1.0)]),
    ]
    assert not any(F.settings_ok(s) for s in bad)
