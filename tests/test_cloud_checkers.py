"""Float64 checkers of the PointCloud2 post steps (SOR and the voxel grid) and the scans that drive the fused
shared-memory chain to its limits.  No GPU here; tests/test_gpu_cloud_limits.py runs the CUDA path through them.

The checkers share no code and no arithmetic with oracle/cloud_oracle.cpp.  They take the cloud BEFORE the step
(the CUDA path's own output of the same nodes with the step switched off -- the projection is pinned to float64 by
test_cloud_semantics.check_projection) and the cloud after it:

  * check_voxel_grid: the cell of a point is floor(float32(x) / float32(voxel)) (the definition's float division);
    the number of cells and every cell's membership are exact, cells come out in the order of their first member,
    the intensity is float32(sum / n) exactly, and each centroid axis lies within 2^-17 m + one float32 ulp of the
    float64 mean of its members.  2^-17 m is the quantisation of the definition's exact integer sums
    (llrintf(v * 65536)); the ulp is the final rounding to float.  So the centroid is NOT held to BASELINE.json's
    1e-6 relative tolerance, which is the projection's: measured on room scans at 0.05 / 0.5 / 4 m voxels the worst
    centroid error is 1.04e-5 m (hypot of both axes), 5.1e-6 relative to the centroid's range.
  * check_sor: the mean distance to the k nearest of the +-16 angular neighbours (all other points when at most 33
    remain) in float64, threshold mean + alpha * std (ddof = 1).  The keep/drop decisions must be the CUDA path's,
    except for points within SOR_MARGIN of the threshold (the definition quantises the means to 2^-16 m and computes
    the distances in float32), and there may only be a few of those.

The mutation tests below plant one fault in the oracle's output and require each checker to reject it."""
import numpy as np
import pytest

from test_gpu_cloud import room_scans

CENTROID_SLACK = 2.0 ** -17  # m: llrintf(v * 65536) rounds every member by at most half of 2^-16
KEYS_PER_QUADRANT = 16384


# ---- the checkers ---------------------------------------------------------------------------------------------------
def voxel_cells(xy, voxel):
    """Cell indices (ix, iy) = floor(float32(x) / float32(voxel)), int64."""
    q = np.asarray(xy, np.float32) / np.float32(voxel)  # float32 division, correctly rounded
    return np.floor(q).astype(np.int64)


def voxel_expectation(base, voxel):
    """Per cell, in the order of their first member: member count, float64 mean x and y, float32 mean intensity."""
    ij = voxel_cells(base[:, :2], voxel)
    _, first, inv = np.unique(ij, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    cell = rank[np.asarray(inv).reshape(-1)]
    n_cells = len(first)
    cnt = np.bincount(cell, minlength=n_cells).astype(np.float64)
    mean = [np.bincount(cell, weights=base[:, a].astype(np.float64), minlength=n_cells) / cnt for a in (0, 1)]
    isum = np.bincount(cell, weights=base[:, 3].astype(np.float64), minlength=n_cells)  # integers: exact
    return cnt, mean, (isum / cnt).astype(np.float32)


def check_voxel_grid(base, got, voxel):
    """base: the cloud before the grid [n, 4]; got: after it.  Returns the worst centroid error (m, per axis)."""
    if base.shape[0] == 0:
        assert got.shape[0] == 0
        return 0.0
    cnt, means, inten = voxel_expectation(base, voxel)
    assert got.shape[0] == len(cnt), (got.shape[0], len(cnt))
    assert (got[:, 3] == inten).all(), "mean intensity"
    assert (got[:, 2] == 0).all()
    worst = 0.0
    for axis, mean in enumerate(means):
        err = np.abs(got[:, axis].astype(np.float64) - mean)
        tol = CENTROID_SLACK + np.spacing(np.abs(mean).astype(np.float32)).astype(np.float64)
        bad = np.flatnonzero(err > tol)
        assert bad.size == 0, (axis, bad[:5], err[bad[:5]], tol[bad[:5]])
        worst = max(worst, float(err.max()))
    return worst


def sor_mean_distances(xy, k):
    """Float64 mean distance of every point to its k nearest among the +-16 angular neighbours (circular; all other
    points when at most 33 remain)."""
    xy = np.asarray(xy, np.float64)
    m = len(xy)
    if m - 1 <= 32:
        d = np.sqrt(((xy[:, None, :] - xy[None, :, :]) ** 2).sum(-1))
        d[np.arange(m), np.arange(m)] = np.inf
        d = np.sort(d, axis=1)[:, : m - 1]
    else:
        offs = np.concatenate([np.arange(-16, 0), np.arange(1, 17)])
        idx = (np.arange(m)[:, None] + offs[None, :]) % m
        d = np.sort(np.sqrt(((xy[idx] - xy[:, None, :]) ** 2).sum(-1)), axis=1)
    return d[:, : min(k, d.shape[1])].mean(axis=1)


def sor_margin(q, thr, alpha):
    """How far from the threshold the definition may decide otherwise than float64: its means are quantised to
    2^-16 m (half of that per point, and the threshold's mean and std move by as much), and its distances are
    float32 sums of at most 32 terms."""
    return 2.0 ** -17 * (2.0 + 1.01 * alpha) + 4e-6 * np.maximum(q, thr)


def kept_mask(base, got):
    """Which points of `base` survive in `got` (which must be a subsequence of it, bit for bit)."""
    bu, gu = base.view(np.uint32), got.view(np.uint32)
    kept = np.zeros(len(base), bool)
    j = 0
    for i in range(len(base)):
        if j < len(got) and (gu[j] == bu[i]).all():
            kept[i] = True
            j += 1
    assert j == len(got), "the SOR output is not a subsequence of its input"
    return kept


def check_sor(base, got, k, alpha):
    """base: the cloud before SOR; got: after it.  Returns the number of points within the margin."""
    m = len(base)
    if m < 2:
        assert (got.view(np.uint32) == base.view(np.uint32)).all()
        return 0
    kept = kept_mask(base, got)
    q = sor_mean_distances(base[:, :2], k)
    thr = q.mean() + alpha * q.std(ddof=1)
    near = np.abs(q - thr) <= sor_margin(q, thr, alpha)
    wrong = np.flatnonzero((kept != (q <= thr)) & ~near)
    assert wrong.size == 0, (wrong[:5], q[wrong[:5]], thr)
    assert near.sum() <= max(3, m // 200), (int(near.sum()), m)
    return int(near.sum())


# ---- case builders --------------------------------------------------------------------------------------------------
def trig_table(O):
    """The float32 cos and sin of every key exactly as the cloud path uses them: the projection of r = 1 m."""
    keys = np.arange(65536)
    pts = O.cloud(O.make_nodes(keys, np.full(65536, 4000), np.zeros(65536, int), 2),
                  O.cloud_params(range_min=0.0, range_max=1e9))
    assert pts.shape[0] == 65536
    return pts[:, 0].copy(), pts[:, 1].copy()


def f32_projection(dist, t):
    """x = float32(dist / 4000) * t in float32, as the definition rounds it."""
    r = np.asarray(dist, np.float32) / np.float32(4000.0)
    return (r * np.asarray(t, np.float32)).astype(np.float32)


def packing_limit_scan(O, seed=5):
    """4096 distinct keys in [0, 16384) at r < 4 m, quality 255: at a 4 m voxel and the new protocol, ONE cell of
    4096 members with an intensity sum of 4096 * 255 = 1,044,480 (the fused chain's 20-bit field holds 1,048,575)."""
    rng = np.random.default_rng(seed)
    keys = np.sort(rng.choice(KEYS_PER_QUADRANT, 4096, replace=False))
    dist = rng.integers(40, 16000, 4096)  # 1 cm .. 3.99975 m
    nodes = O.make_nodes(keys, dist, np.full(4096, 255), 2)
    return np.roll(nodes, -int(rng.integers(0, 4096)))


def corner_scan(O, quadrant):
    """One cell of 4096 points in quadrant `quadrant`: the leader (smallest key) 1 cm from the sensor, at the cell's
    corner at the origin; the 4095 others 3.995 m out along the quadrant's first half, at the opposite edge of the cell
    on the dominant axis.  At a 4 m voxel the per-leader sum of 16.16 fixed-point deltas on that axis passes 1.0e9
    (2^31 = 2.147e9 is where the fused chain's int accumulators wrap)."""
    base = quadrant * KEYS_PER_QUADRANT
    rel = np.unique(np.linspace(182, 8010, 4095).astype(np.int64))  # 1 .. 44 degrees into the quadrant
    assert len(rel) == 4095
    r = 3.995 / np.cos(rel * (2 * np.pi / 65536))
    keys = np.concatenate([[base + 1], base + rel])
    dist = np.concatenate([[40], np.rint(r * 4000.0).astype(np.int64)])
    nodes = O.make_nodes(keys, dist, (np.arange(4096) * 7) % 256, 2)
    return np.roll(nodes, -1234)


def dominant_axis(quadrant):
    return quadrant & 1  # x in quadrants 0 and 2, y in 1 and 3


def fix16(v):
    """llrintf(v * 65536) for float32 v (the scale is exact; rint rounds half to even like llrintf)."""
    return np.rint(np.asarray(v, np.float32).astype(np.float64) * 65536.0).astype(np.int64)


BOUNDARY_VOXELS = (0.05, 0.1, 0.25, 1.0 / 3.0)
ULPS = (-3, -2, -1, 0, 1, 2, 3)
TINY_KEYS = (0, KEYS_PER_QUADRANT, 2 * KEYS_PER_QUADRANT, 3 * KEYS_PER_QUADRANT)  # a coordinate within 1e-7 of 0


def ulps_from_integer(q):
    """(ulps of float32 q away from the nearest integer in magnitude, that integer); + = larger magnitude."""
    q = np.asarray(q, np.float32)
    n = np.rint(q).astype(np.float32)
    return np.abs(q).view(np.int32).astype(np.int64) - np.abs(n).view(np.int32).astype(np.int64), n


def boundary_scan(O, trig, voxel, per_class=24, seed=0):
    """Points whose float32 x / voxel or y / voxel is an exact integer, or 1-3 ulps either side of one, with both signs,
    each key at most once (<= 4096 nodes: the fused chain serves it); plus the keys where cos or sin is within 1e-7
    of zero, at several ranges.  Found by search over (key, dist) with the exact float32 trig table."""
    rng = np.random.default_rng(seed)
    v32 = np.float32(voxel)
    used = set()
    keys, dists = [], []
    for t_axis in trig:
        cand_k, cand_d, cand_u, cand_s = [], [], [], []
        for n in (1, 2, 3, 7, 19, 60):
            ks = np.flatnonzero(np.abs(t_axis) >= 0.05)
            target = n * float(voxel) / np.abs(t_axis[ks].astype(np.float64)) * 4000.0
            ok = target < 30.0 * 4000.0
            ks, target = ks[ok], target[ok]
            for dd in (-1, 0, 1):
                d = np.rint(target).astype(np.int64) + dd
                x = f32_projection(d, t_axis[ks])
                u, near = ulps_from_integer(x / v32)
                sel = (np.abs(u) <= 3) & (near != 0)
                cand_k.append(ks[sel]); cand_d.append(d[sel]); cand_u.append(u[sel]); cand_s.append(np.sign(x[sel]))
        ck, cd, cu, cs = (np.concatenate(a) for a in (cand_k, cand_d, cand_u, cand_s))
        for s in (-1.0, 1.0):
            for u in ULPS:
                idx = np.flatnonzero((cu == u) & (cs == s))
                rng.shuffle(idx)
                taken = 0
                for i in idx:
                    if taken == per_class:
                        break
                    if int(ck[i]) in used:
                        continue
                    used.add(int(ck[i]))
                    keys.append(int(ck[i]))
                    dists.append(int(cd[i]))
                    taken += 1
    for j, k in enumerate(TINY_KEYS):
        if k not in used:
            keys.append(k)
            dists.append(400 * (j + 1) + int(seed))
    order = np.argsort(keys)
    keys, dists = np.asarray(keys)[order], np.asarray(dists)[order]
    assert len(keys) <= 4096
    nodes = O.make_nodes(keys, dists, rng.integers(0, 256, len(keys)), 2)
    return np.roll(nodes, -int(rng.integers(0, len(keys))))


def window_scan(O, m, seed, stride=400):
    """A room scan of `stride` nodes of which exactly m survive the window (the others unmeasured)."""
    nodes = room_scans(O, 1, stride, seed)[0]
    nodes["dist_mm_q2"] = np.clip(nodes["dist_mm_q2"], 4000, 100000)  # every node inside [0.15, 40] m
    rng = np.random.default_rng(seed)
    off = np.ones(stride, bool)
    off[rng.choice(stride, m, replace=False)] = False
    nodes["dist_mm_q2"][off] = 0
    return nodes


SOR_WINDOW_COUNTS = (2, 3, 32, 33, 34, 35)  # around the all-others / window switch (m - 1 <= 32)


def spike_scan(O, n, seed):
    """A circular wall 2.5 m around the sensor, keys evenly spaced, with isolated spikes (single points 0.5-2 m further
    out, 16-90 points apart).  On the wall the 8 nearest neighbours of a point are its +-4 in angle; only the points
    whose +-4 hold a spike find a nearer one further out, so in a warp only some lanes do."""
    rng = np.random.default_rng(seed)
    keys = (np.arange(n) * 65536) // n
    dist = np.full(n, 10000)
    pos = np.cumsum(rng.integers(16, 90, n // 16))
    pos = pos[pos < n]
    dist[pos] += rng.integers(2000, 8000, len(pos))
    nodes = O.make_nodes(keys, dist, rng.integers(0, 256, n), 2)
    return np.roll(nodes, -int(rng.integers(0, n)))


def later_group_lanes(xy):
    """Per point of an angle-ordered cloud (window form): does one of its neighbours at +-5..16 lie nearer than the
    8th nearest of its neighbours at +-1..4?  (sor_mean_win8's merge of a later group changes the result only then.)"""
    xy = np.asarray(xy, np.float64)
    m = len(xy)
    near = np.concatenate([np.arange(-4, 0), np.arange(1, 5)])
    far = np.concatenate([np.arange(-16, -4), np.arange(5, 17)])
    dn = np.sqrt(((xy[(np.arange(m)[:, None] + near) % m] - xy[:, None]) ** 2).sum(-1)).max(1)
    df = np.sqrt(((xy[(np.arange(m)[:, None] + far) % m] - xy[:, None]) ** 2).sum(-1)).min(1)
    return df < dn


def cpu_cloud(O, nodes, **kw):
    return O.cloud(nodes, O.cloud_params(**kw))


# ---- the checkers accept the definition -----------------------------------------------------------------------------
@pytest.mark.parametrize("voxel", [0.05, 0.5, 4.0])
def test_voxel_checker_accepts_the_definition(oracle, voxel):
    worst = 0.0
    for seed in range(4):
        nodes = room_scans(oracle, 1, 3200, 100 + seed)[0]
        base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
        got = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0, voxel_size=voxel)
        worst = max(worst, check_voxel_grid(base, got, voxel))
    # the 2^-17 slack is needed (a bare float32 ulp would reject the definition) and not much looser than the truth
    assert 2.0 ** -18 < worst <= CENTROID_SLACK + 2.0 ** -21


@pytest.mark.parametrize("k", [1, 8, 17, 32])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 2.5])
def test_sor_checker_accepts_the_definition(oracle, k, alpha):
    for seed in range(2):
        nodes = room_scans(oracle, 1, 3200, 300 + seed)[0]
        base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
        got = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0, sor_k=k, sor_alpha=alpha)
        check_sor(base, got, k, alpha)
    for nodes in [window_scan(oracle, m, 40 + m) for m in SOR_WINDOW_COUNTS] + [spike_scan(oracle, 3200, 7)]:
        base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
        check_sor(base, cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0, sor_k=k, sor_alpha=alpha), k, alpha)


# ---- ... and reject one planted fault ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def voxel_case(oracle):
    nodes = room_scans(oracle, 1, 3200, 17)[0]
    base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
    got = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0, voxel_size=0.05)
    check_voxel_grid(base, got, 0.05)
    return nodes, base, got


def test_voxel_checker_rejects_a_centroid_moved_by_2_pow_minus_16(voxel_case):
    _, base, got = voxel_case
    cnt, means, _ = voxel_expectation(base, 0.05)
    for r in (int(np.argmax(cnt == 1)), int(np.argmax(cnt)), len(cnt) - 1):  # one member, the most, the last cell
        for axis in (0, 1):
            bad = got.copy()
            step = 2.0 ** -16 if got[r, axis] >= means[axis][r] else -(2.0 ** -16)  # away from the float64 mean
            bad[r, axis] = np.float32(np.float64(got[r, axis]) + step)
            with pytest.raises(AssertionError):
                check_voxel_grid(base, bad, 0.05)


def test_voxel_checker_rejects_two_cells_swapped(voxel_case):
    _, base, got = voxel_case
    bad = got.copy()
    bad[[10, 11]] = got[[11, 10]]
    with pytest.raises(AssertionError):
        check_voxel_grid(base, bad, 0.05)


def test_voxel_checker_rejects_an_intensity_off_by_one(voxel_case):
    _, base, got = voxel_case
    bad = got.copy()
    bad[20, 3] += 1.0
    with pytest.raises(AssertionError):
        check_voxel_grid(base, bad, 0.05)


def test_voxel_checker_rejects_a_point_moved_to_the_neighbouring_cell(oracle, voxel_case):
    """The output of the definition for the same nodes but one range a quarter millimetre or two different, which
    carries that point across a cell boundary: the checker is given the unchanged input."""
    nodes, base, got = voxel_case
    order = np.argsort(nodes["angle_z_q14"], kind="stable")
    measured = order[(nodes["dist_mm_q2"][order] >= 600)]
    assert len(measured) == len(base)
    cells = voxel_cells(base[:, :2], 0.05)
    for p in np.argsort(np.abs(base[:, 0] / np.float32(0.05) - np.rint(base[:, 0] / np.float32(0.05)))):
        for dd in (-2, -1, 1, 2):
            moved = nodes.copy()
            moved["dist_mm_q2"][measured[p]] = int(moved["dist_mm_q2"][measured[p]]) + dd
            b2 = cpu_cloud(oracle, moved, range_min=0.15, range_max=40.0)
            c2 = voxel_cells(b2[p : p + 1, :2], 0.05)[0]
            if c2[0] != cells[p, 0] and c2[1] == cells[p, 1]:
                bad = cpu_cloud(oracle, moved, range_min=0.15, range_max=40.0, voxel_size=0.05)
                assert np.abs(b2[:, :2] - base[:, :2]).max() < 1e-3  # nothing else moved, and that one < 1 mm
                with pytest.raises(AssertionError):
                    check_voxel_grid(base, bad, 0.05)
                return
    pytest.fail("no point within two range steps of a cell boundary")


def test_sor_checker_rejects_one_decision_flipped(oracle):
    nodes = room_scans(oracle, 1, 3200, 301)[0]
    base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
    got = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0, sor_k=8, sor_alpha=1.0)
    check_sor(base, got, 8, 1.0)
    kept = kept_mask(base, got)
    q = sor_mean_distances(base[:, :2], 8)
    thr = q.mean() + q.std(ddof=1)
    clear = np.abs(q - thr) > 10 * sor_margin(q, thr, 1.0)
    drop_one = kept.copy()
    drop_one[np.flatnonzero(kept & clear)[len(got) // 2]] = False  # a kept point well below the threshold dropped
    keep_one = kept.copy()
    keep_one[np.flatnonzero(~kept & clear)[0]] = True  # an outlier well above it kept
    for mask in (drop_one, keep_one):
        with pytest.raises(AssertionError):
            check_sor(base, base[mask], 8, 1.0)


# ---- the case builders make what the GPU tests claim ----------------------------------------------------------------
def test_packing_limit_scan_is_one_cell_at_the_20_bit_limit(oracle):
    nodes = packing_limit_scan(oracle)
    assert len(np.unique(nodes["angle_z_q14"])) == 4096 and nodes["angle_z_q14"].max() < KEYS_PER_QUADRANT
    base = cpu_cloud(oracle, nodes, range_min=0.0, range_max=40.0, is_new_protocol=1)
    assert base.shape[0] == 4096
    assert (voxel_cells(base[:, :2], 4.0) == 0).all()
    assert int(base[:, 3].astype(np.int64).sum()) == 1044480 < 2 ** 20
    got = cpu_cloud(oracle, nodes, range_min=0.0, range_max=40.0, is_new_protocol=1, voxel_size=4.0)
    assert got.shape[0] == 1 and got[0, 3] == 255.0


@pytest.mark.parametrize("quadrant", [0, 1, 2, 3])
def test_corner_scan_has_deltas_past_1e9(oracle, quadrant):
    nodes = corner_scan(oracle, quadrant)
    assert len(np.unique(nodes["angle_z_q14"])) == 4096
    base = cpu_cloud(oracle, nodes, range_min=0.0, range_max=40.0)
    assert base.shape[0] == 4096
    cells = voxel_cells(base[:, :2], 4.0)
    want = [[0, 0], [-1, 0], [-1, -1], [0, -1]][quadrant]
    assert (cells == want).all()
    assert np.abs(base[0, :2]).max() < 0.0101  # the leader (first in angle order) sits at the origin corner
    a = dominant_axis(quadrant)
    delta = int((fix16(base[1:, a]) - fix16(base[0, a])).sum())
    assert 1.0e9 <= abs(delta) < 2 ** 31, delta
    assert (delta > 0) == (quadrant in (0, 1))


@pytest.mark.parametrize("voxel", BOUNDARY_VOXELS)
def test_boundary_scan_hits_every_ulp_class(oracle, voxel):
    trig = trig_table(oracle)
    nodes = boundary_scan(oracle, trig, voxel)
    assert len(np.unique(nodes["angle_z_q14"])) == len(nodes) <= 4096
    base = cpu_cloud(oracle, nodes, range_min=0.0, range_max=40.0)
    assert base.shape[0] == len(nodes)
    v32 = np.float32(voxel)
    shortcut_wrong = 0
    for axis in (0, 1):
        q = base[:, axis] / v32
        u, near = ulps_from_integer(q)
        hit = (np.abs(u) <= 3) & (near != 0)
        for s in (-1, 1):
            for k in ULPS:
                assert ((u == k) & (near != 0) & (np.sign(q) == s)).sum() >= 5, (axis, s, k)
        # the fused kernel's first guess x * RN(1 / voxel) is this close to an integer for (nearly) every one of them,
        # so its floor_div falls back to the division
        q0 = (base[:, axis] * (np.float32(1.0) / v32)).astype(np.float32)
        fallback = np.abs(q0 - np.rint(q0)).astype(np.float32) <= np.abs(q0) * np.float32(4e-7)
        assert fallback[hit & (np.abs(u) <= 2)].all() and fallback[hit].mean() > 0.9
        shortcut_wrong += int((np.floor(q0) != np.floor(q)).sum())
    if voxel == 1.0 / 3.0:  # (1 / voxel is exact in float for the others) the guess alone would pick the wrong cell
        assert shortcut_wrong > 0
    keys = np.sort(nodes["angle_z_q14"])  # = the order of `base`: every node is kept
    sel = np.isin(keys, TINY_KEYS)
    assert sel.sum() == len(TINY_KEYS)
    assert (np.abs(base[sel, :2]).min(axis=1) < 3e-6).all()
    assert base[keys == KEYS_PER_QUADRANT, 0][0] < 0  # cos(float32(pi / 2)) = -4.4e-8: x sits just left of 0


def test_window_scans_leave_m_points(oracle):
    for m in SOR_WINDOW_COUNTS:
        assert cpu_cloud(oracle, window_scan(oracle, m, 40 + m), range_min=0.15, range_max=40.0).shape[0] == m


def test_spike_scan_gives_mixed_warps(oracle):
    nodes = spike_scan(oracle, 3200, 7)
    base = cpu_cloud(oracle, nodes, range_min=0.15, range_max=40.0)
    later = later_group_lanes(base[:, :2])
    per_warp = np.add.reduceat(later.astype(int), np.arange(0, len(later), 32))
    lanes = np.minimum(32, len(later) - np.arange(0, len(later), 32))
    mixed = (per_warp > 0) & (per_warp < lanes)
    assert mixed.sum() >= 20 and (per_warp == 0).sum() >= 5
