"""Session nodes (rpl_*_stream_nodes[_dev], CapsuleStreamSession.nodes / nodes_dev): after a push, the node buffer
RealLidarDriver::grab_scan_data would return for every scan that push published, ascended and packed on the device.
Every comparison is bit for bit on nodes, counts and statuses: the buffers concatenated over the pushes of a stream
split into pieces against oracle/scan_oracle.cpp (O.ascend, stable tie rule) on the restated scans of the whole stream
(the restatements the LaserScan session tests hold the sessions to), and against rpl_scan_batch_dev's nodes_out on those
same scans."""
import numpy as np
import pytest

from test_gpu_capsule_stream import _scans
from test_gpu_stream_cloud import KINDS, MAX_SCANS, PARAMS, REV_NODES, Feed, cloud_rows, hq_stream, splits

pytestmark = pytest.mark.gpu

OK, FAIL = 0, 0x80008001


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def u64(a):
    return np.ascontiguousarray(a).view(np.uint64)


def rows_of(bufs, status, sps, n, max_scans):
    """per stream, the buffers of one nodes call: [(status, node bits)]; unused slots are empty with status OK"""
    rows = []
    for s in range(n):
        k = min(int(sps[s]), max_scans)
        for j in range(k, max_scans):
            assert len(bufs[s * max_scans + j]) == 0 and status[s * max_scans + j] == OK, (s, j)
        rows.append([(int(status[s * max_scans + j]), u64(bufs[s * max_scans + j]).tobytes()) for j in range(k)])
    return rows


def expected_rows(R, O, ctx, restated, ascend=True):
    """per stream, the definition's buffers of the whole stream's scans; the ascended ones checked against
    rpl_scan_batch_dev's nodes_out on the same scans"""
    rows = []
    for scans, lens, k in restated:
        rows.append([])
        for j in range(k):
            h = scans[j, : lens[j]]
            rc, buf = O.ascend(h, stable=True) if ascend else (OK, h)
            rows[-1].append((rc, u64(buf).tobytes()))
    if ascend:
        nodes = np.concatenate([s[:k] for s, _, k in restated])
        counts = np.concatenate([l[:k] for _, l, k in restated]).astype(np.uint32)
        flat = [r for row in rows for r in row]
        for at in range(0, len(flat), ctx.max_scans):
            hi = min(at + ctx.max_scans, len(flat))
            got = ctx.scan_batch(np.ascontiguousarray(nodes[at:hi]).view(R.NODE_DTYPE), counts[at:hi],
                                 R.scan_params(*PARAMS), emit_nodes=True)
            assert [(int(got["status"][j]), u64(got["nodes"][j, : counts[at + j]]).tobytes())
                    for j in range(hi - at)] == flat[at:hi]
    return rows


def check_packing(p, ns):
    """offsets: the exclusive scan of the even-rounded counts; total: the end of the last buffer"""
    counts, offs = p["node_counts"].astype(np.uint64), p["node_offsets"]
    even = (counts + 1) & ~np.uint64(1)
    assert (offs == np.concatenate([[0], np.cumsum(even)[:-1]]).astype(np.uint64)).all()
    used = np.nonzero(counts)[0]
    assert p["total_nodes"] == (int(offs[used[-1]] + counts[used[-1]]) if len(used) else 0)
    assert len(offs) == ns


def run(R, feed, sess, pieces, stride, kw):
    """pushes the pieces with host pushes, one host nodes call after each (kw None: none); LaserScans and buffers per
    stream"""
    n = len(pieces[0])
    scans, rows = [[] for _ in range(n)], [[] for _ in range(n)]
    for push in pieces:
        out = feed.push(sess, push, stride)
        for s, row in enumerate(_scans(out, n, sess.max_scans)):
            scans[s] += row
        if kw is not None:
            p = sess.nodes(packed=True, **kw)
            check_packing(p, n * sess.max_scans)
            bufs = [p["nodes"][o: o + c] for o, c in zip(p["node_offsets"].tolist(), p["node_counts"].tolist())]
            for s, row in enumerate(rows_of(bufs, p["status"], out["scans_per_stream"], n, sess.max_scans)):
                rows[s] += row
    return scans, rows


@pytest.mark.parametrize("kind,ans", KINDS)
def test_pushes_give_the_whole_streams_buffers(R, oracle, kind, ans):
    """every format and session kind, each stream split into three pushes at its own points (some pieces empty: the
    stream idles in that push), max_nodes 8192: ascended, passed through, and a per-stream mix"""
    feed = Feed(R, oracle, kind, ans)
    n, max_nodes = 8, 8192
    streams = [feed.data(s, REV_NODES[s % len(REV_NODES)] + (s // len(REV_NODES))) for s in range(n)]
    pieces = splits(np.random.default_rng(ans + len(kind)), streams, 3)
    pieces[1][2], pieces[2][2] = pieces[1][2][:0], np.concatenate([pieces[1][2], pieces[2][2]])  # stream 2 idles once
    stride = max(len(p) for push in pieces for p in push)
    ctx = R.Context(0, max_nodes, 256)
    mask = np.arange(n) % 3 != 1
    got = {}
    for name, kw in (("asc", dict(apply_ascend=True)), ("raw", dict(apply_ascend=False)),
                     ("mix", dict(apply_ascend=False, per_stream=mask)), ("none", None)):
        with feed.session(ctx, n, stride, max_nodes) as sess:
            got[name] = run(R, feed, sess, pieces, stride, kw)
    assert got["asc"][0] == got["none"][0] == got["raw"][0] == got["mix"][0]  # the pushes' own outputs
    restated = [feed.restated(d, max_nodes) for d in streams]
    lens = np.concatenate([l[:k] for _, l, k in restated])
    assert (lens > 4096).any() and (lens <= 4096).any() and (lens % 2 == 1).any()
    asc, raw = expected_rows(R, oracle, ctx, restated), expected_rows(R, oracle, ctx, restated, ascend=False)
    assert got["asc"][1] == asc
    assert got["raw"][1] == raw
    assert got["mix"][1] == [asc[s] if mask[s] else raw[s] for s in range(n)]
    assert all(len(r) >= 2 for r in asc) and asc != raw
    ctx.close()


def crafted_stream(O, revs):
    """HQ capsules carrying the given revolutions (arrays of NODE_DTYPE whose first node has the start flag) behind a
    leading one, then the start of one more"""
    lead = revs[0][:1].repeat(10)
    lead["flag"][1:] = 2
    nodes = np.concatenate([lead] + list(revs) + [revs[0][:1]])
    n = (len(nodes) + 95) // 96
    pad = np.zeros(n * 96 - len(nodes), O.NODE_DTYPE)
    pad["angle_z_q14"], pad["dist_mm_q2"], pad["flag"] = 7, 400, 2
    nodes = np.concatenate([nodes, pad])
    payload = np.zeros((n, 781), np.uint8)
    payload[:, 9:9 + 768] = nodes.view(np.uint8).reshape(n, 768)
    return O.seal_capsules(0x83, payload)


def rev(O, rng, n, measured=True, dup=0):
    """one revolution of n nodes with rising distinct keys; `dup` nodes repeat their predecessor's key; unmeasured
    nodes sprinkled in (all of them with measured=False)"""
    r = np.zeros(n, O.NODE_DTYPE)
    r["angle_z_q14"] = np.sort(rng.choice(65536, n, replace=False))
    if dup:
        at = rng.choice(np.arange(1, n), dup, replace=False)
        r["angle_z_q14"][at] = r["angle_z_q14"][at - 1]
    r["dist_mm_q2"] = rng.integers(1, 160000, n) if measured else 0
    if measured:
        r["dist_mm_q2"][rng.random(n) < 0.1] = 0
        r["dist_mm_q2"][rng.integers(0, n)] = 1234
    r["quality"] = rng.integers(0, 256, n)
    r["flag"] = 2
    r["flag"][0] = 1
    return r


@pytest.mark.parametrize("max_nodes", [64, 8192])
def test_revolution_shapes(R, oracle, max_nodes):
    """lengths 1, 2, odd (the next view starts on an odd node), max_nodes and above it (the capacity rule comes first),
    an all-unmeasured revolution (OPERATION_FAIL, buffer unchanged), many duplicate final keys (the general kernel);
    max_nodes 8192: revolutions of 4097-8192 nodes"""
    O, rng = oracle, np.random.default_rng(max_nodes)
    big = [4097, 8191, 8192, 8200] if max_nodes == 8192 else [63, 64, 65, 90]
    shapes = [[(1, {}), (2, {}), (33, {}), (big[0], {}), (40, dict(measured=False)), (big[1], {})],
              [(big[2], {}), (big[3], {}), (50, dict(dup=30)), (5, {}), (big[0], dict(dup=big[0] // 2))],
              [(7, dict(measured=False)), (1, dict(measured=False)), (21, {}), (34, dict(dup=1))]]
    feed = Feed(R, O, "framed", 0x83)
    streams = [crafted_stream(O, [rev(O, rng, m, **kw) for m, kw in sh]) for sh in shapes]
    stride = max(len(d) for d in streams)
    ctx = R.Context(0, 8192, 64)
    with feed.session(ctx, len(streams), stride, max_nodes, 8) as sess:  # 8 scan slots: 7 revolutions at most
        _, rows = run(R, feed, sess, [streams], stride, dict(apply_ascend=True))
        _, raw = run(R, feed, sess, [[d[:0] for d in streams]], stride, dict(apply_ascend=False))
        assert all(r == [] for r in raw)  # a push that published nothing
    restated = [feed.restated(d, max_nodes) for d in streams]
    exp = expected_rows(R, O, ctx, restated)
    assert rows == exp
    flat = [r for row in exp for r in row]
    assert sum(rc == FAIL for rc, _ in flat) == 4 and {len(b) // 8 for _, b in flat} >= {1, 2, 33, max_nodes}
    ctx.close()


def dev_nodes(torch, sess, capacity=None, stream=None, **kw):
    """nodes_dev into fresh device buffers with a canary behind them"""
    ns = sess.n_streams * sess.max_scans
    cap = ns * sess.max_nodes if capacity is None else capacity
    nodes = torch.full((cap + 64,), -7, dtype=torch.int64, device="cuda")
    offs = torch.full((ns,), -1, dtype=torch.int64, device="cuda")
    counts = torch.full((ns,), -1, dtype=torch.int32, device="cuda")
    status = torch.full((ns,), -1, dtype=torch.int32, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    sess.nodes_dev(nodes.data_ptr(), cap, offs.data_ptr(), counts.data_ptr(), status.data_ptr(), total.data_ptr(),
                   stream=None if stream is None else stream.cuda_stream, **kw)
    torch.cuda.synchronize()
    return dict(nodes=nodes.cpu().numpy().view(np.uint64), node_offsets=offs.cpu().numpy().view(np.uint64),
                node_counts=counts.cpu().numpy().view(np.uint32), status=status.cpu().numpy().view(np.uint32),
                total_nodes=int(total.cpu().numpy()[0]))


def packed_rows(p, sps, n, max_scans):
    bufs = [p["nodes"][o: o + c] for o, c in zip(p["node_offsets"].tolist(), p["node_counts"].tolist())]
    return rows_of(bufs, p["status"], sps, n, max_scans)


def test_host_and_device_chunking_differ(R, oracle):
    """chunk_host (2 streams: large capsule strides) != chunk_dev (3 streams: the context's max_scans): a host push
    followed by nodes_dev, a push_dev followed by the host nodes; a per-stream mask across the chunks"""
    import torch

    feed = Feed(R, oracle, "framed", 0x83)
    n, max_nodes, stride = 7, 8192, 8000
    streams = [hq_stream(oracle, 3, REV_NODES[s % 4] + s, 900 + s, dup_share=0.001) for s in range(n)]
    pieces = splits(np.random.default_rng(5), streams, 2)
    ctx = R.Context(0, max_nodes, 3 * MAX_SCANS)
    mask = np.array([1, 0, 1, 1, 0, 0, 1], np.uint8)
    kws = [dict(apply_ascend=True), dict(per_stream=mask), dict(apply_ascend=False)]
    got = [[[] for _ in range(n)] for _ in kws]
    with feed.session(ctx, n, stride, max_nodes) as sess:
        out = feed.push(sess, pieces[0], stride)  # host push: chunks of 2
        for i, kw in enumerate(kws):
            p = dev_nodes(torch, sess, **kw)
            check_packing(p, n * MAX_SCANS)
            assert (p["nodes"][p["total_nodes"]:] == np.uint64(2**64 - 7)).all()  # nothing at or past the total
            for s, row in enumerate(packed_rows(p, out["scans_per_stream"], n, MAX_SCANS)):
                got[i][s] += row
        buf, cnt = feed.pack(pieces[1], stride)  # device push: chunks of 3
        NS = n * MAX_SCANS
        d_buf, d_cnt = torch.from_numpy(buf).cuda(), torch.from_numpy(cnt.view(np.int32)).cuda()
        r, it = torch.zeros((NS, max_nodes), device="cuda"), torch.zeros((NS, max_nodes), device="cuda")
        bc, inc = torch.zeros(NS, dtype=torch.int32, device="cuda"), torch.zeros(NS, device="cuda")
        sps = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        sess.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                      bc.data_ptr(), inc.data_ptr(), sps.data_ptr())
        ctx.synchronize()
        for i, kw in enumerate(kws):
            p = sess.nodes(packed=True, **kw)
            check_packing(p, NS)
            for s, row in enumerate(packed_rows(p, sps.cpu().numpy().view(np.uint32), n, MAX_SCANS)):
                got[i][s] += row
    restated = [feed.restated(d, max_nodes) for d in streams]
    asc, raw = expected_rows(R, oracle, ctx, restated), expected_rows(R, oracle, ctx, restated, ascend=False)
    assert got[0] == asc and got[2] == raw
    assert got[1] == [asc[s] if mask[s] else raw[s] for s in range(n)]
    ctx.close()


def test_capacity_repeat_calls_reset_and_bad_calls(R, oracle):
    import torch

    feed = Feed(R, oracle, "framed", 0x84)
    n, max_nodes = 4, 8192
    streams = [feed.data(s, REV_NODES[s]) for s in range(n)]
    stride = max(len(d) for d in streams)
    ctx = R.Context(0, max_nodes, 64)
    prm = R.cloud_params(range_min=0.15, range_max=40.0, sor_k=8, voxel_size=0.05)
    ns = n * MAX_SCANS
    with feed.session(ctx, n, stride, max_nodes) as sess:
        big = torch.zeros(ns * max_nodes, dtype=torch.int64, device="cuda")
        tab = torch.zeros(4 * ns + 4, dtype=torch.int64, device="cuda")
        a = [big.data_ptr(), ns * max_nodes, tab.data_ptr(), tab.data_ptr() + 8 * ns, tab.data_ptr() + 12 * ns,
             tab.data_ptr() + 16 * ns]
        for call in (lambda: sess.nodes(), lambda: sess.nodes_dev(*a)):
            with pytest.raises(R.RplError) as e:  # no push yet
                call()
            assert e.value.code == R.RESULT_INVALID_DATA
        out = feed.push(sess, streams, stride)
        sps = out["scans_per_stream"]
        cloud = sess.cloud(prm)
        msgs = sess.laserscan_msgs(R.scan_params(*PARAMS))
        first = sess.nodes(packed=True)
        rows = packed_rows(first, sps, n, MAX_SCANS)
        assert sum(len(r) for r in rows) >= 2 * n
        total = first["total_nodes"]
        # the cloud and message calls give what they gave before the nodes call; the nodes call repeats itself
        again = sess.cloud(prm)
        assert cloud_rows(again, sps, n, MAX_SCANS) == cloud_rows(cloud, sps, n, MAX_SCANS)
        assert sess.laserscan_msgs(R.scan_params(*PARAMS)) == msgs
        sess.reset()
        assert packed_rows(sess.nodes(packed=True), sps, n, MAX_SCANS) == rows
        assert packed_rows(dev_nodes(torch, sess), sps, n, MAX_SCANS) == rows
        # exactly enough room; then one node short: nothing written, counts 0, the total still reported
        fit = dev_nodes(torch, sess, capacity=total)
        assert packed_rows(fit, sps, n, MAX_SCANS) == rows and (fit["nodes"][total:] == np.uint64(2**64 - 7)).all()
        short = dev_nodes(torch, sess, capacity=total - 1)
        assert short["total_nodes"] == total and (short["node_counts"] == 0).all() and (short["status"] == OK).all()
        assert (short["nodes"] == np.uint64(2**64 - 7)).all()
        assert (short["node_offsets"] == first["node_offsets"]).all()
        hbuf = np.zeros(total - 1, R.NODE_DTYPE)
        u64(hbuf)[:] = 0x0505
        h = sess.nodes(packed=True, nodes=hbuf)
        assert h["result"] == R.capi.RESULT_INSUFFICIENT_MEMORY and h["total_nodes"] == total
        assert (h["node_counts"] == 0).all() and (u64(hbuf) == 0x0505).all()
        with pytest.raises(R.RplError) as e:
            sess.nodes(nodes=hbuf)
        assert e.value.code == R.capi.RESULT_INSUFFICIENT_MEMORY
        exact = sess.nodes(packed=True, nodes=np.zeros(total, R.NODE_DTYPE))
        assert exact["result"] == OK and packed_rows(exact, sps, n, MAX_SCANS) == rows
        for i in (0, 2, 3, 4, 5):  # null pointers
            bad = list(a)
            bad[i] = None
            with pytest.raises(R.RplError) as e:
                sess.nodes_dev(*bad)
            assert e.value.code == R.RESULT_INVALID_DATA
        for i, by in ((0, 8), (2, 4), (3, 2), (4, 2), (5, 4)):  # misaligned device buffers
            bad = list(a)
            bad[i] += by
            with pytest.raises(R.RplError) as e:
                sess.nodes_dev(*bad)
            assert e.value.code == R.RESULT_INVALID_DATA
        assert packed_rows(sess.nodes(packed=True), sps, n, MAX_SCANS) == rows  # still there
        buf, cnt = feed.pack(streams, stride)
        cnt[1] = stride + 1
        with pytest.raises(R.RplError):  # a failed push leaves no nodes to take
            sess.push(buf, cnt, R.scan_params(*PARAMS))
        with pytest.raises(R.RplError) as e:
            sess.nodes()
        assert e.value.code == R.RESULT_INVALID_DATA
    restated = [feed.restated(d, max_nodes) for d in streams]
    assert rows == expected_rows(R, oracle, ctx, restated)
    ctx.close()


def test_side_stream_then_next_push(R, oracle):
    """nodes_dev on a side torch stream, then a push_dev on another stream before anyone waits: the buffers are the
    first push's"""
    import torch

    feed = Feed(R, oracle, "dense", 0x85)
    n, max_nodes = 6, 4096
    streams = [feed.data(s, REV_NODES[s % 4]) for s in range(n)]
    pieces = splits(np.random.default_rng(3), streams, 2)
    stride = max(len(p) for push in pieces for p in push)
    ctx = R.Context(0, 8192, 256)
    side, other = torch.cuda.Stream(), torch.cuda.Stream()
    NS = n * MAX_SCANS
    with feed.session(ctx, n, stride, max_nodes) as sess:
        out = feed.push(sess, pieces[0], stride)
        nodes = torch.zeros(NS * max_nodes, dtype=torch.int64, device="cuda")
        offs, total = torch.zeros(NS, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
        counts, status = torch.zeros(NS, dtype=torch.int32, device="cuda"), torch.zeros(NS, dtype=torch.int32, device="cuda")
        buf, cnt = feed.pack(pieces[1], stride)
        d_buf, d_cnt = torch.from_numpy(buf).cuda(), torch.from_numpy(cnt.view(np.int32)).cuda()
        r, it = torch.zeros((NS, max_nodes), device="cuda"), torch.zeros((NS, max_nodes), device="cuda")
        bc, inc = torch.zeros(NS, dtype=torch.int32, device="cuda"), torch.zeros(NS, device="cuda")
        sps = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        sess.nodes_dev(nodes.data_ptr(), NS * max_nodes, offs.data_ptr(), counts.data_ptr(), status.data_ptr(),
                       total.data_ptr(), stream=side.cuda_stream)
        sess.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                      bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=other.cuda_stream)
        torch.cuda.synchronize()
        p = dict(nodes=nodes.cpu().numpy().view(np.uint64), node_offsets=offs.cpu().numpy().view(np.uint64),
                 node_counts=counts.cpu().numpy().view(np.uint32), status=status.cpu().numpy().view(np.uint32))
        got = packed_rows(p, out["scans_per_stream"], n, MAX_SCANS)
        bufs, st = sess.nodes()
        for s, row in enumerate(rows_of(bufs, st, sps.cpu().numpy().view(np.uint32), n, MAX_SCANS)):
            got[s] += row
    restated = [feed.restated(d, max_nodes) for d in streams]
    assert got == expected_rows(R, oracle, ctx, restated)
    ctx.close()
