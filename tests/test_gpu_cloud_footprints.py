"""Footprints in the clouds on the device (rpl_cloud_footprint_batch_dev, RPL_CLOUD_PER_STREAM_FOOTPRINTS) against the
definition of tests/test_cloud_footprints_oracle.py.

The stateless call must be the definition bit for bit on every route of the chain.  A session's flagged clouds must be,
stream by stream, what the stateless call gives on the same scan's nodes (the session's grabbed node buffers, not
ascended) with that stream's footprint in the cloud's frame: the footprint as set, or for an inverted stream under
RPL_CLOUD_PER_STREAM the mirrored footprint (vertices (x, -y) at pose (px, -py, -yaw)), whose scan-frame vertices are
exactly (u, -v)."""
import math

import numpy as np
import pytest

from oracle import scan_footprint_oracle as FP
from test_cloud_footprints_oracle import cloud_with_footprint, random_scan
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_push_msgs import lidar_settings, make_session, pieces_for
from test_gpu_stream_stamps import _streams

pytestmark = pytest.mark.gpu
FILL = np.float32(-7.25)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


def as_rpl(R, fp):
    """the binding's footprint of an oracle footprint"""
    polys = [[(float(fp.x[p][k]), float(fp.y[p][k])) for k in range(fp.n_vertices[p])] for p in range(4)
             if fp.n_vertices[p]]
    inv = [fp.invert[p] for p in range(4) if fp.n_vertices[p]]
    return R.scan_footprint(polys, inv, pose=(fp.pose_x, fp.pose_y, fp.pose_yaw))


def mirrored(R, f):
    """the cloud-frame footprint of an inverted stream: its scan-frame vertices are (u, -v)"""
    polys = [[(f.x[p][k], -f.y[p][k]) for k in range(f.n_vertices[p])] for p in range(4) if f.n_vertices[p]]
    inv = [f.invert[p] for p in range(4) if f.n_vertices[p]]
    return R.scan_footprint(polys, inv, pose=(f.pose_x, -f.pose_y, -f.pose_yaw))


def star(rng, k, cx, cy, r0, r1):
    ang = np.sort(rng.uniform(0, 2 * math.pi, k))
    rad = rng.uniform(r0, r1, k)
    return [(cx + a * math.cos(t), cy + a * math.sin(t)) for a, t in zip(rad, ang)]


def fleet_footprints(R, n):
    """a body with the lidar at a corner, a box, a region of interest, four 16-vertex polygons, an L, none"""
    rng = np.random.default_rng(7)
    table = [
        R.scan_footprint([[(-1.5, -1.0), (1.5, -1.0), (1.5, 1.0), (-1.5, 1.0)]], pose=(1.5, 1.0, math.radians(45))),
        R.scan_footprint([[(-2.0, -1.0), (2.0, -1.0), (2.0, 1.0), (-2.0, 1.0)]]),
        R.scan_footprint([[(-1.0, -4.0), (6.0, 0.0), (-1.0, 4.0)]], invert=[1], pose=(-0.5, 0.2, 0.3)),
        R.scan_footprint([star(rng, 16, *rng.uniform(-2, 2, 2), 0.5, 5.0) for _ in range(4)], invert=[0, 1, 0, 0],
                         pose=(0.3, -0.4, 2.0)),
        R.scan_footprint([[(0.0, 0.0), (4.0, 0.0), (4.0, 2.0), (2.0, 2.0), (2.0, 4.0), (0.0, 4.0)]],
                         pose=(1.0, 1.0, -2.5)),
        R.scan_footprint(),
    ]
    return [table[s % len(table)] for s in range(n)]


def stateless(R, torch, ctx, scans, stride, params, fp, fn="cloud_footprint_batch_dev"):
    """(counts, xyzi rows) of the stateless call over the node arrays `scans`"""
    n = len(scans)
    buf = np.zeros((n, stride), R.NODE_DTYPE)
    cnt = np.zeros(n, np.uint32)
    for j, s in enumerate(scans):
        buf[j, : len(s)] = s
        cnt[j] = len(s)
    d_nodes = torch.from_numpy(buf.view(np.int64)).cuda()
    d_cnt = torch.from_numpy(cnt.view(np.int32)).cuda()
    xyzi = torch.full((n, stride, 4), float(FILL), dtype=torch.float32, device="cuda")
    pc = torch.zeros(n, dtype=torch.int32, device="cuda")
    if fn == "cloud_batch_dev":
        ctx.cloud_batch_dev(d_nodes.data_ptr(), d_cnt.data_ptr(), n, stride, params, xyzi.data_ptr(), pc.data_ptr())
    else:
        ctx.cloud_footprint_batch_dev(d_nodes.data_ptr(), d_cnt.data_ptr(), n, stride, params, fp, xyzi.data_ptr(),
                                      pc.data_ptr())
    ctx.synchronize()
    pc = pc.cpu().numpy().view(np.uint32)
    xyzi = xyzi.cpu().numpy()
    return pc, [xyzi[j, : pc[j]].tobytes() for j in range(n)]


CHAINS = [dict(), dict(sor_k=8, sor_alpha=1.0), dict(voxel_size=0.05), dict(sor_k=4, sor_alpha=0.5, voxel_size=0.2)]


@pytest.mark.parametrize("n_nodes,stride", [(700, 1024), (3000, 4096), (6500, 8192)])
def test_stateless_is_the_definition(R, oracle, torch, n_nodes, stride):
    rng = np.random.default_rng(n_nodes)
    ctx = R.Context(0, stride, 8)
    scans = [random_scan(oracle, rng, int(rng.integers(n_nodes // 2, n_nodes + 1)), dup_share=0.01 * (j % 2))
             for j in range(8)]
    for t in range(3):
        fp = FP.footprint([star(rng, int(rng.integers(3, 17)), *rng.uniform(-3, 3, 2), 0.3, 4.0)
                           for _ in range(int(rng.integers(1, 5)))], [int(rng.random() < 0.2) for _ in range(4)],
                          pose=(*rng.uniform(-1, 1, 2), float(rng.uniform(-4, 4))))
        for kw in CHAINS:
            p = oracle.cloud_params(0.15, 40.0, 0.0, is_new_protocol=1, **kw)
            exp = [cloud_with_footprint(oracle, s, p, fp) for s in scans]
            for flags in (0, R.CLOUD_NO_FUSED):
                prm = R.cloud_params(0.15, 40.0, 0.0, is_new_protocol=1, flags=flags, **kw)
                pc, rows = stateless(R, torch, ctx, scans, stride, prm, as_rpl(R, fp))
                assert pc.tolist() == [len(e) for e in exp], (t, kw, flags)
                assert rows == [e.tobytes() for e in exp], (t, kw, flags)
    ctx.close()


def test_null_or_empty_footprint_is_cloud_batch_dev(R, oracle, torch):
    rng = np.random.default_rng(5)
    ctx = R.Context(0, 4096, 6)
    scans = [random_scan(oracle, rng, 3000, dup_share=0.01) for _ in range(6)]
    for kw in CHAINS:
        for flags in (0, R.CLOUD_NO_FUSED):
            prm = R.cloud_params(0.15, 40.0, 0.0, is_new_protocol=1, flags=flags, **kw)
            n0 = ctx.launch_count
            ref = stateless(R, torch, ctx, scans, 4096, prm, None, fn="cloud_batch_dev")
            per_call = ctx.launch_count - n0
            for fp in (None, R.scan_footprint(), R.scan_footprint(pose=(3.0, -2.0, 1.0))):
                n1 = ctx.launch_count
                got = stateless(R, torch, ctx, scans, 4096, prm, fp)
                assert got[0].tolist() == ref[0].tolist() and got[1] == ref[1]
                assert ctx.launch_count - n1 == per_call
    ctx.close()


def test_refusals(R, torch):
    ctx = R.Context(0, 1024, 2)
    d = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    a = d.data_ptr()
    prm = R.cloud_params()
    bad = [R.scan_footprint([[(0, 0), (1, 0)]]), R.scan_footprint([[(0, 0), (1001, 0), (0, 1)]]),
           R.scan_footprint([[(0, 0), (1, 0), (0, 1)]], pose=(float("nan"), 0, 0)),
           R.scan_footprint([[(0, 0), (1, 0), (0, 1)]], pose=(0, -1000.5, 0))]
    for fp in bad:
        with pytest.raises(R.RplError) as e:
            ctx.cloud_footprint_batch_dev(a, a, 1, 16, prm, fp, a, a)
        assert e.value.code == R.RESULT_INVALID_DATA
    for args in [(0, a, a, a), (a, 0, a, a), (a, a, 0, a), (a, a, a, 0)]:
        with pytest.raises(R.RplError) as e:
            ctx.cloud_footprint_batch_dev(args[0], args[1], 1, 16, prm, R.scan_footprint(), args[2], args[3])
        assert e.value.code == R.RESULT_INVALID_DATA
    ctx.close()


def session_expected(R, torch, ctx, sess, n, ms, max_nodes, flags, table, fps, lidars):
    """per stream and slot, (count, bytes) of the stateless call on that scan's nodes"""
    bufs, _ = sess.nodes(apply_ascend=False)
    exp = []
    for s in range(n):
        scans = [bufs[s * ms + k] for k in range(ms)]
        newp = lidars[s].is_new_protocol if (lidars and flags & R.CLOUD_PER_STREAM) else 1
        e = table[s] if flags & R.CLOUD_PER_STREAM_CHAIN else None
        if e is not None and not e.enabled:
            exp.append(None)
            continue
        kw = dict(voxel_size=e.voxel_size, sor_k=e.sor_k, sor_alpha=e.sor_alpha) if e else dict(sor_k=8, sor_alpha=1.0,
                                                                                                   voxel_size=0.05)
        rmin, rmax, imin = (e.range_min, e.range_max or sess_rmax(n)[s], e.intensity_min) if e else (0.15, 30.0, 0.0)
        prm = R.cloud_params(rmin, rmax, imin, is_new_protocol=newp, flags=flags & R.CLOUD_NO_FUSED, **kw)
        fp = fps[s]
        if lidars and flags & R.CLOUD_PER_STREAM and lidars[s].inverted:
            fp = mirrored(R, fp)
        if not (flags & R.CLOUD_PER_STREAM_FOOTPRINTS):
            fp = None
        pc, rows = stateless(R, torch, ctx, scans, max_nodes, prm, fp)
        exp.append((pc.tolist(), rows))
    return exp


def sess_rmax(n):
    return np.linspace(0.5, 40.0, n).astype(np.float32)


def cloud_table(R, n):
    table = [R.cloud_settings(0.2, 0.0, 0.0), R.cloud_settings(0.15, 0.0, 0.0, voxel_size=0.05),
             R.cloud_settings(0.15, 30.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0),
             R.cloud_settings(0.15, 40.0, 0.0, voxel_size=0.05, enabled=False),
             R.cloud_settings(0.1, 40.0, 0.0, voxel_size=0.001, sor_k=4, sor_alpha=0.5),
             R.cloud_settings(0.3, 25.0, 2.0, sor_k=12, sor_alpha=2.0), R.cloud_settings(0.15, 0.0, 1.0, sor_k=8)]
    return [table[s % len(table)] for s in range(n)]


def session_params(R, flags):
    return R.cloud_params(0.15, 30.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0, is_new_protocol=1, flags=flags)


def check_calls(R, torch, ctx, sess, n, ms, max_nodes, flags, table, fps, lidars, push_msgs=None):
    exp = session_expected(R, torch, ctx, sess, n, ms, max_nodes, flags, table, fps, lidars)
    prm = session_params(R, flags)
    got = sess.cloud(prm)
    xyzi = torch.full((n * ms, max_nodes, 4), float(FILL), dtype=torch.float32, device="cuda")
    pcd = torch.zeros(n * ms, dtype=torch.int32, device="cuda")
    sess.cloud_dev(prm, xyzi.data_ptr(), pcd.data_ptr())
    ctx.synchronize()
    dev = dict(point_counts=pcd.cpu().numpy().view(np.uint32), xyzi=xyzi.cpu().numpy())
    msgs = sess.cloud_msgs(prm)
    for s in range(n):
        for out in (got, dev):
            pc = out["point_counts"][s * ms:(s + 1) * ms]
            if exp[s] is None:
                assert (pc == 0).all(), s
                continue
            assert pc.tolist() == exp[s][0], (s, flags)
            assert [out["xyzi"][s * ms + k, : pc[k]].tobytes() for k in range(ms)] == exp[s][1], (s, flags)
        for k in range(ms):
            m, c = msgs[s * ms + k], int(got["point_counts"][s * ms + k])
            if m is not None:
                assert m[len(m) - 1 - 16 * c: len(m) - 1] == got["xyzi"][s * ms + k, :c].tobytes(), (s, k)
    if push_msgs is not None:
        assert push_msgs == msgs
    return sum(int(c > 0) for c in got["point_counts"])


FLAGSETS = ["fp", "fp+chain", "fp+per", "fp+chain+per", "fp+chain+nofused", "none+chain"]


def flags_of(R, name):
    f = R.CLOUD_PER_STREAM_FOOTPRINTS if name.startswith("fp") else 0
    f |= R.CLOUD_PER_STREAM_CHAIN if "chain" in name else 0
    f |= R.CLOUD_PER_STREAM if "per" in name else 0
    f |= R.CLOUD_NO_FUSED if "nofused" in name else 0
    return f


def push_pair(R, torch, ctx, A, B, n, ms, mx, buf, cnt, sp, cprm, dev):
    """one push on A (push / push_dev) and the same push as push_cloud_msgs[_dev] on B: B's messages per slot"""
    if not dev:
        A.push(buf, cnt, sp)
        return B.push_cloud_msgs(buf, cnt, cprm)[0]
    d = torch.device("cuda", 0)
    NS = n * ms
    tb, tc = torch.from_numpy(buf).to(d), torch.from_numpy(cnt.view(np.int32)).to(d)
    rg, it = (torch.empty((NS, mx), dtype=torch.float32, device=d) for _ in range(2))
    bc, sps = torch.empty(NS, dtype=torch.int32, device=d), torch.empty(n, dtype=torch.int32, device=d)
    inc = torch.empty(NS, dtype=torch.float32, device=d)
    A.push_dev(tb.data_ptr(), tc.data_ptr(), sp, rg.data_ptr(), it.data_ptr(), bc.data_ptr(), inc.data_ptr(),
               sps.data_ptr())
    cap = NS * ((288 + 116 + 16 * mx + 1 + 15) // 16 * 16)
    store = torch.zeros(cap, dtype=torch.uint8, device=d)
    offs, total = torch.zeros(NS, dtype=torch.int64, device=d), torch.zeros(1, dtype=torch.int64, device=d)
    sizes, tsps = torch.zeros(NS, dtype=torch.int32, device=d), torch.zeros(n, dtype=torch.int32, device=d)
    B.push_cloud_msgs_dev(tb.data_ptr(), tc.data_ptr(), cprm, 0, store.data_ptr(), cap, offs.data_ptr(),
                          sizes.data_ptr(), total.data_ptr(), tsps.data_ptr())
    ctx.synchronize()
    m, o, z = store.cpu().numpy(), offs.cpu().numpy().view(np.uint64), sizes.cpu().numpy().view(np.uint32)
    return [bytes(m[a: a + b]) if b else None for a, b in zip(o.tolist(), z.tolist())]


def run_sessions(R, torch, ctx, kind, ans, n, ms, mx, stride, pieces, fps, types=None):
    """A (pushes, cloud calls) and B (push_cloud_msgs) fed the pieces, host and device pushes alternating, the flag sets
    cycling; after every push each of A's cloud calls and B's messages against the stateless call.  Returns the number
    of clouds compared."""
    A = make_session(R, ctx, kind, ans, n, stride, mx, ms, types)
    B = make_session(R, ctx, kind, ans, n, stride, mx, ms, types)
    lid = lidar_settings(R, n)
    table = cloud_table(R, n)
    for x in (A, B):
        x.set_frames(["base_scan"] * n, sess_rmax(n))
        x.set_lidars(lid)
        x.set_clouds(table)
        with pytest.raises(R.RplError) as e:  # flagged before set_scan_footprints
            x.cloud(session_params(R, R.CLOUD_PER_STREAM_FOOTPRINTS))
        assert e.value.code == R.RESULT_INVALID_DATA
        x.set_scan_footprints(fps)
    seen = 0
    for t, push in enumerate(pieces):
        flags = flags_of(R, FLAGSETS[t % len(FLAGSETS)])
        if kind == "framed":
            buf = np.zeros((n, stride, A.capsule_bytes), np.uint8)
        else:
            buf = np.full((n, stride), 0xEE, np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s in range(n):
            buf[s, : len(push[s])] = push[s]
            cnt[s] = len(push[s])
        sp = R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM if flags & R.CLOUD_PER_STREAM else 0)
        pm = push_pair(R, torch, ctx, A, B, n, ms, mx, buf, cnt, sp, session_params(R, flags), dev=t % 2 == 1)
        seen += check_calls(R, torch, ctx, A, n, ms, mx, flags, table, fps, lid, pm)
        if t == 1:  # a masked footprint change between pushes
            mask = np.zeros(n, np.uint8)
            mask[1::2] = 1
            new = fleet_footprints(R, n + 1)[1:]
            for x in (A, B):
                x.set_scan_footprints(new, mask)
            fps = [new[s] if mask[s] else fps[s] for s in range(n)]
    A.close()
    B.close()
    return seen


def mixed_pieces(O, types, rng):
    streams = [_streams(O, t, 1, 9500 + s)[0].reshape(-1) for s, t in enumerate(types)]
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams])
    return pieces, max(1, max(len(x) for push in pieces for x in push))


CASES = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + \
        [("bytes", a) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)] + [("mixed", 0)]


@pytest.mark.parametrize("kind,ans", CASES)
def test_sessions_are_the_stateless_call(R, oracle, torch, kind, ans):
    n, ms, mx = 7, 3, 4096
    rng = np.random.default_rng(ans + 17 * (kind == "bytes"))
    types = None
    if kind == "mixed":
        types = [(0x81, 0x82, 0x83, 0x84, 0x85, 0x86)[s % 6] for s in range(n)]
        pieces, stride = mixed_pieces(oracle, types, rng)
        kind = "bytes"
    else:
        _, pieces, stride = pieces_for(oracle, kind, ans, n, 9100 + ans, rng)
    ctx = R.Context(0, mx, n * ms)
    assert run_sessions(R, torch, ctx, kind, ans, n, ms, mx, stride, pieces, fleet_footprints(R, n), types) > n
    ctx.close()


def test_several_chunks_per_push(R, oracle, torch):
    """23 streams in device chunks of 3 and host chunks of 4; the streams 3..7 have no polygons, so one device chunk
    (3..5) and one host chunk (4..7) run without the pass between chunks that run it"""
    n, ms, mx = 23, 3, 4096
    streams = [c.reshape(-1) for c in _streams(oracle, 0x82, n, 1700)]
    rng = np.random.default_rng(31)
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams])
    stride = (16 << 20) // 5 + 1  # 16 MiB // stride = 4 streams per host chunk
    ctx = R.Context(0, mx, 3 * ms)  # 3 streams per device chunk
    fps = [R.scan_footprint() if 3 <= s <= 7 else f for s, f in enumerate(fleet_footprints(R, n))]
    assert run_sessions(R, torch, ctx, "bytes", 0x82, n, ms, mx, stride, pieces, fps) > n
    ctx.close()


def test_no_polygons_no_extra_launch(R, oracle, torch):
    n, ms, mx = 6, 3, 4096
    rng = np.random.default_rng(3)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x84, n, 9300, rng)
    ctx = R.Context(0, mx, n * ms)
    A = make_session(R, ctx, "framed", 0x84, n, stride, mx, ms)
    A.set_frames(["f"] * n, sess_rmax(n))
    A.set_clouds(cloud_table(R, n))
    A.set_scan_footprints([R.scan_footprint(pose=(1.0, 2.0, 0.5))] * n)
    for push in pieces:
        buf = np.zeros((n, stride, A.capsule_bytes), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s in range(n):
            buf[s, : len(push[s])] = push[s]
            cnt[s] = len(push[s])
        A.push(buf, cnt, R.scan_params(1, 0, 0, 1))
        for base in (0, R.CLOUD_PER_STREAM_CHAIN, R.CLOUD_NO_FUSED):
            outs, counts = [], []
            for f in (base, base | R.CLOUD_PER_STREAM_FOOTPRINTS):
                n0 = ctx.launch_count
                outs.append(A.cloud(session_params(R, f)))
                counts.append(ctx.launch_count - n0)
            assert counts[0] == counts[1]
            assert outs[0]["point_counts"].tolist() == outs[1]["point_counts"].tolist()
            assert outs[0]["xyzi"].tobytes() == outs[1]["xyzi"].tobytes()
    A.close()
    ctx.close()


@pytest.mark.parametrize("mode_a", [0, 1], ids=["mode_b", "mode_a"])
def test_end_to_end_nothing_inside_the_body(R, oracle, torch, mode_a):
    n, ms, mx = 4, 3, 4096
    rng = np.random.default_rng(20 + mode_a)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x83, n, 9400, rng)
    ctx = R.Context(0, mx, n * ms)
    A = make_session(R, ctx, "framed", 0x83, n, stride, mx, ms)
    lid = [R.lidar_settings(1, mode_a, s % 2) for s in range(n)]
    body = [(-3.0, -2.0), (3.0, -2.0), (3.0, 2.0), (-3.0, 2.0)]
    fps = [R.scan_footprint([body], pose=(3.0, 2.0, math.radians(45 + 30 * s))) for s in range(n)]
    A.set_frames(["f"] * n, np.full(n, 40.0, np.float32))
    A.set_lidars(lid)
    A.set_scan_filters([R.scan_filter_settings()] * n)
    A.set_scan_footprints(fps)
    removed = 0
    for push in pieces:
        buf = np.zeros((n, stride, A.capsule_bytes), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s in range(n):
            buf[s, : len(push[s])] = push[s]
            cnt[s] = len(push[s])
        out = A.push(buf, cnt, R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM | R.FLAG_PER_STREAM_FILTERS))
        prm = R.cloud_params(0.15, 40.0, 0.0, flags=R.CLOUD_PER_STREAM | R.CLOUD_PER_STREAM_FOOTPRINTS)
        cl = A.cloud(prm)
        plain = A.cloud(R.cloud_params(0.15, 40.0, 0.0, flags=R.CLOUD_PER_STREAM))
        for s in range(n):
            fpo = FP.footprint([body], pose=(fps[s].pose_x, fps[s].pose_y, fps[s].pose_yaw))
            (u, v, _), = FP.scan_frame(fpo)
            for k in range(min(int(out["scans_per_stream"][s]), ms)):
                j = s * ms + k
                c = int(cl["point_counts"][j])
                x, y = cl["xyzi"][j, :c, 0], cl["xyzi"][j, :c, 1]
                assert not FP.inside(u, -v if lid[s].inverted else v, x, y).any(), (s, k)
                removed += int(plain["point_counts"][j]) - c
                M = int(out["beam_counts"][j])
                r = out["ranges"][j, :M]
                fin = np.isfinite(r)
                bx, by = FP.beam_points(np.where(fin, r, 0), out["angle_increment"][j])
                assert not (FP.inside(u, v, bx, by) & fin).any(), (s, k)
    assert removed > 0
    A.close()
    ctx.close()
