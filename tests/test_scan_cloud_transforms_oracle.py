"""CPU checks of the definition of projected clouds in a target frame (tests/scan_cloud_transform_oracle.py): R against
scipy, the points against float64, the identity and disabled entries against P, an upside-down mount against an
inverted lidar, the limits, and the field table of every channel set."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import scan_cloud_transform_oracle as SCT
from oracle import cdr_oracle as CDR
from oracle import scan_cloud_oracle as SC

NAN, INF = float("nan"), float("inf")
EPS = float(np.finfo(np.float32).eps)


def _quats(rng, n):
    axis = [(1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (-1, 0, 0, 0), (0, 0, 0, -1),
            (math.sqrt(0.5), 0, 0, math.sqrt(0.5)), (0, 0, math.sin(0.3), math.cos(0.3))]
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    # non-unit ones inside the limit: |d - 1| up to 0.9e-3
    q *= np.sqrt(1.0 + rng.uniform(-0.9e-3, 0.9e-3, (n, 1)))
    return [tuple(map(float, a)) for a in axis] + [tuple(map(float, v)) for v in q]


def _scan(ranges, inc=0.0175, ti=1e-4, frame="laser_frame", range_max=12.0):
    r = np.asarray(ranges, np.float32)
    return dict(sec=12, nanosec=34, frame_id=frame, angle_min=0.0, angle_increment=np.float32(inc),
                time_increment=np.float32(ti), range_min=np.float32(0.15), range_max=np.float32(range_max), ranges=r,
                intensities=np.arange(r.size, dtype=np.float32))


def _ranges(rng, M):
    r = rng.uniform(0.15, 11.0, M).astype(np.float32)
    r[rng.random(M) < 0.1] = np.float32(NAN)
    r[rng.random(M) < 0.05] = np.float32(INF)
    return r


def test_rotation_is_scipys_to_float_rounding():
    rng = np.random.default_rng(1)
    for q in _quats(rng, 200):
        want = Rotation.from_quat(q).as_matrix()
        R64 = SCT.rotation_matrix(q)
        assert np.abs(R64 - want).max() < 1e-12
        R, _ = SCT.transform_rows(q, (0, 0, 0))
        assert R.dtype == np.float32 and np.abs(R.astype(np.float64) - want[:, :2]).max() <= EPS


def test_points_are_float64_R_p_plus_t_within_ulps():
    rng = np.random.default_rng(2)
    for q in _quats(rng, 40):
        t = rng.uniform(-50, 50, 3)
        M = int(rng.integers(1, 8193))
        r = _ranges(rng, M)
        inc = np.float32(2 * np.pi / M)
        base = SC.project(SC.params(0), r, r, inc, 0.0, 0.15, 12.0)
        got = SCT.project(SC.params(0), r, r, inc, 0.0, 0.15, 12.0, SCT.transform(t, q))
        p = base.view("<f4").reshape(-1, 3).astype(np.float64)
        X = got.view("<f4").reshape(-1, 3).astype(np.float64)
        want = p @ Rotation.from_quat(q).as_matrix().T + t
        scale = np.abs(p[:, :1]) + np.abs(p[:, 1:2]) + np.abs(t)
        assert (np.abs(X - want) <= 4 * EPS * scale).all()


@pytest.mark.parametrize("ch", range(16))
def test_identity_is_P_bit_for_bit(ch):
    rng = np.random.default_rng(3 + ch)
    for M in (1, 2, 360, 3200, 8192):
        r = _ranges(rng, M)
        for inc in (np.float32(2 * np.pi / M), np.float32(-2 * np.pi / M)):
            s = _scan(r, inc=inc)
            base = SC.project(SC.params(ch), r, s["intensities"], inc, 1e-4, 0.15, 12.0)
            got = SCT.project(SC.params(ch), r, s["intensities"], inc, 1e-4, 0.15, 12.0, SCT.transform())
            assert got.tobytes() == base.tobytes()
            assert SCT.P(SC.params(ch), s, SCT.transform(), "laser_frame") == SC.P(SC.params(ch), s)


@pytest.mark.parametrize("ch", range(32))
def test_disabled_entry_is_P(ch):
    rng = np.random.default_rng(40 + ch)
    r = _ranges(rng, 720)
    s = _scan(r)
    off = SCT.transform((3, 4, 5), (0, 0, 1, 0), enabled=False)
    got = SCT.P(SC.params(ch), s, off, "base_link")
    base = SC.P(SC.params(ch & 0xF), s)
    if not ch & SCT.VIEWPOINT:
        assert got == base
    msg, ref = CDR.parse_pointcloud2(got), CDR.parse_pointcloud2(base)
    assert msg["frame_id"] == "laser_frame" and msg["width"] == ref["width"]
    rec, rrec = SC.cloud_records(msg), SC.cloud_records(ref)
    for name in rrec.dtype.names:
        assert rec[name].tobytes() == rrec[name].tobytes()
    if ch & SCT.VIEWPOINT:
        for name in SCT.VIEWPOINT_FIELDS:
            assert (rec[name].view(np.uint32) == 0).all()


def test_upside_down_mount_is_the_inverted_lidar(oracle):
    """roll pi on a non-inverted stream gives (x, -y, 0); so does the inverted stream's beam M-1-i under identity"""
    O = oracle
    p = SC.params(SC.INDEX)
    roll = SCT.transform(rotation=(1.0, 0.0, 0.0, 0.0))
    for nodes in (O.dummy_scan(1), O.synth_batch(5, 1, 3200, 4)[0], O.synth_batch(9, 1, 8000, 0)[0]):
        _, asc = O.ascend(nodes)
        h0, r0, i0 = O.publish(asc, O.scan_params(0, 0, 0, 1, 40.0, 0.1))
        h1, r1, i1 = O.publish(asc, O.scan_params(0, 0, 1, 1, 40.0, 0.1))
        M = h0.beam_count
        assert h1.beam_count == M and M > 0
        a = SCT.project(p, r0[:M], i0[:M], h0.angle_increment, 0, h0.range_min, h0.range_max, roll)
        b = SCT.project(p, r1[:M], i1[:M], h1.angle_increment, 0, h1.range_min, h1.range_max, SCT.transform())
        A, B = a.view("<f4").reshape(-1, 4)[:, :3], b.view("<f4").reshape(-1, 4)[:, :3]
        ia, ib = a.view("<u4").reshape(-1, 4)[:, 3], b.view("<u4").reshape(-1, 4)[:, 3]
        assert a.shape[0] == b.shape[0] > 0
        at = {int(i): k for k, i in enumerate(ib)}
        for k, i in enumerate(ia):
            j = at[M - 1 - int(i)]
            tol = 1e-6 * max(1.0, float(np.abs(A[k]).max()))
            assert np.abs(A[k] - B[j]).max() <= tol
        assert (A[:, 2].view(np.uint32) == 0).all() and (B[:, 2].view(np.uint32) == 0).all()


def _limit_cases():
    """(entry, frame, ok): both sides of every bound"""
    T = SCT.transform
    lim = 1e-3
    ok_q = (0.0, 0.0, 0.0, math.sqrt(1 + lim * 0.999))
    out = [(T(), "base_link", True), (T(), "", True), (T(), "a" * 255, True), (T(), "a" * 256, False),
           (T(rotation=ok_q), "b", True), (T(rotation=(0.0, 0.0, 0.0, math.sqrt(1 + lim * 1.001))), "b", False),
           (T(rotation=(0.0, 0.0, 0.0, math.sqrt(1 - lim * 0.999))), "b", True),
           (T(rotation=(0.0, 0.0, 0.0, math.sqrt(1 - lim * 1.001))), "b", False),
           (T(rotation=(0.0, 0.0, 0.0, 0.0)), "b", False)]
    for k in range(3):
        for v, good in ((1000.0, True), (-1000.0, True), (1000.0001, False), (-1000.0001, False), (NAN, False),
                        (INF, False)):
            t = [0.0, 0.0, 0.0]
            t[k] = v
            out.append((T(t), "b", good))
    for k in range(4):
        for v in (NAN, INF, -INF):
            q = [0.0, 0.0, 0.0, 1.0]
            q[k] = v
            out.append((T(rotation=q), "b", False))
    # a disabled entry is not read
    out.append((T((NAN, 0, 0), (0, 0, 0, 0), enabled=False), None, True))
    return out


def test_limits_both_sides():
    for e, frame, good in _limit_cases():
        assert SCT.transform_ok(e, frame) == good, (e, frame)


def test_channel_rules():
    for ch in range(32):
        assert SCT.params_ok(SC.params(ch), True)
        assert SCT.params_ok(SC.params(ch), False) == (ch < 16)
        assert SCT.params_ok(SC.params(ch | SCT.PER_STREAM_TRANSFORMS), True)
    for bad in (0x20, 0x40, 0x80, 0x200):
        assert not SCT.params_ok(SC.params(bad), True)
    assert not SCT.params_ok(SC.params(0x13, NAN), True)


@pytest.mark.parametrize("ch", range(32))
def test_field_table_and_point_step(ch):
    names = ["intensity", "index", "distances", "stamps"]
    types = [SC.FLOAT32, SC.INT32, SC.FLOAT32, SC.FLOAT32]
    present = [k for k in range(4) if ch >> k & 1]
    want = [("x", 0, SC.FLOAT32, 1), ("y", 4, SC.FLOAT32, 1), ("z", 8, SC.FLOAT32, 1)] + \
        [(names[k], 12 + 4 * j, types[k], 1) for j, k in enumerate(present)]
    if ch & SCT.VIEWPOINT:
        want += [(n, 12 + 4 * len(present) + 4 * j, SC.FLOAT32, 1) for j, n in enumerate(("vp_x", "vp_y", "vp_z"))]
    assert SCT.fields(ch) == want
    assert SCT.point_step(ch) == 12 + 4 * len(present) + 12 * bool(ch & SCT.VIEWPOINT)
    t = SCT.transform((1.5, -2.0, 0.25), (0.1, 0.2, 0.3, math.sqrt(1 - 0.14)))
    s = _scan([1.0, NAN, 2.0, 3.0], ti=2.5e-4)
    msg = CDR.parse_pointcloud2(SCT.P(SC.params(ch), s, t, "base_link"))
    assert msg["fields"] == want and msg["point_step"] == SCT.point_step(ch)
    assert msg["frame_id"] == "base_link" and (msg["sec"], msg["nanosec"]) == (12, 34)
    assert msg["width"] == 3 and msg["row_step"] == 3 * msg["point_step"] and msg["is_dense"] == 1
    rec = SC.cloud_records(msg)
    if ch & SCT.VIEWPOINT:
        vp = np.float32([1.5, -2.0, 0.25])
        for k, n in enumerate(SCT.VIEWPOINT_FIELDS):
            assert (rec[n] == vp[k]).all()
