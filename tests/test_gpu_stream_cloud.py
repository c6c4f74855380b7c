"""Session clouds (rpl_*_stream_cloud[_dev], CapsuleStreamSession.cloud / cloud_dev): after a push, the PointCloud2
chain over exactly the scans that push published, read in place from the session's arenas.  Every comparison is bit
for bit on xyzi and point counts: the clouds concatenated over the pushes of a stream split into pieces against
oracle/cloud_oracle.cpp (O.cloud) on the restated scans of the whole stream (the restatements the LaserScan session
tests hold the sessions to), and against rpl_cloud_batch_dev on those same scans.  Sessions of max_nodes 8192 meet
revolutions of 4097-8192 nodes, which the fused kernel hands to the general kernel; duplicate measured keys and odd
revolution lengths (views starting on odd nodes) are part of the streams."""
import numpy as np
import pytest

from test_capsule_bytes_pieces import restated_scans as bytes_restated
from test_capsule_oracle_vs_ref import make_capsules
from test_capsule_stream_pieces import restated_scans as capsule_restated
from test_decode_oracle_vs_ref import make_stream
from test_gpu_capsule_stream import _scans
from test_gpu_cloud_exchange import dev_bytes
from test_normal_stream_pieces import normal_stream, restated_scans as normal_restated

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
NODES_PER_CAP = {0x82: 32, 0x83: 96, 0x84: 96, 0x85: 40, 0x86: 64}
REV_NODES = (2950, 5801, 7303, 4097)  # what a lidar delivers, and revolutions the fused kernel hands on at max_nodes 8192
MAX_SCANS = 24  # a damaged stream publishes short scans while the decoder resynchronises
WINDOW = dict(range_min=0.15, range_max=40.0)
SOR = dict(sor_k=8, sor_alpha=1.0)
VOXEL = dict(voxel_size=0.05)
SETTINGS = [dict(), SOR, VOXEL, dict(**SOR, **VOXEL)]


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def hq_stream(O, n_revs, rev_nodes, seed, dup_share=0.0):
    """HQ capsules of revolutions of rev_nodes nodes (angles rising, flag bit 0 on each revolution's first node); with
    dup_share, that share of the nodes repeats its predecessor's key"""
    rng = np.random.default_rng(seed)
    n = int(n_revs * rev_nodes / 96) + 2
    m = n * 96
    pos = (np.arange(m) + int(rng.integers(0, rev_nodes))) % rev_nodes
    key = (pos * 65536 // rev_nodes + rng.integers(0, 3, m)) & 0xFFFF
    dup = np.nonzero(rng.random(m) < dup_share)[0]
    dup = dup[dup > 0]
    key[dup] = key[dup - 1]
    nodes = np.zeros(m, O.NODE_DTYPE)
    nodes["angle_z_q14"] = key
    nodes["dist_mm_q2"] = rng.integers(0, 40000 * 4, m)
    nodes["dist_mm_q2"][rng.random(m) < 0.05] = 0
    nodes["quality"] = rng.integers(0, 256, m)
    start = pos == 0
    nodes["flag"] = start.astype(np.uint8) | ((~start).astype(np.uint8) << 1)
    payload = rng.integers(0, 256, (n, 781), dtype=np.uint8)
    payload[:, 9:9 + 768] = nodes.view(np.uint8).reshape(n, 768)
    return O.seal_capsules(0x83, payload)


def capsule_stream(O, ans, n_revs, rev_nodes, seed):
    """[n, capsule bytes]: about n_revs revolutions of about rev_nodes nodes"""
    if ans == 0x83:
        return hq_stream(O, n_revs, rev_nodes, seed, dup_share=0.001)
    cpr = rev_nodes / NODES_PER_CAP[ans]
    n = int(n_revs * cpr) + 3
    if ans == 0x85:
        return make_stream(O, n, cpr, seed=seed)
    return make_capsules(O, ans, n, cpr, seed=seed)


class Feed:
    """One session kind: framed capsules, the dense session, 0x81 bytes or the raw bytes of a capsule format"""

    def __init__(self, R, O, kind, ans):
        self.R, self.O, self.kind, self.ans = R, O, kind, ans

    def data(self, s, rev_nodes, n_revs=4):
        seed = 4000 + 17 * s + self.ans
        if self.kind == "normal":
            return normal_stream(n_revs * rev_nodes, seed, nodes_per_rev=rev_nodes, bad=False)
        caps = capsule_stream(self.O, self.ans, n_revs, rev_nodes, seed)
        if self.kind != "bytes":
            return caps
        b = caps.reshape(-1)  # a few noise runs for the sync-byte search
        rng = np.random.default_rng(seed)
        at = np.sort(rng.choice(len(b), 3, replace=False))
        parts = np.split(b, at)
        noise = [rng.integers(0, 0xA0, int(rng.integers(1, 40)), dtype=np.uint8) for _ in at]
        return np.concatenate([p for pair in zip(parts, noise + [parts[-1][:0]]) for p in pair])

    def session(self, ctx, n, stride, max_nodes, max_scans=MAX_SCANS):
        R = self.R
        if self.kind == "normal":
            return R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans)
        if self.kind == "bytes":
            return R.CapsuleByteStreamSession(ctx, self.ans, n, stride, max_nodes, max_scans)
        if self.kind == "dense":
            return R.DenseStreamSession(ctx, n, stride, max_nodes, max_scans)
        return R.CapsuleStreamSession(ctx, self.ans, n, stride, max_nodes, max_scans)

    def pack(self, push, stride):
        """one push's pieces (per stream) -> (buffer, counts) in the session's input layout"""
        unit = push[0].shape[1:]
        buf = np.zeros((len(push), stride) + unit, np.uint8)
        cnt = np.zeros(len(push), np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        return buf, cnt

    def push(self, sess, push, stride):
        buf, cnt = self.pack(push, stride)
        return sess.push(buf, cnt, self.R.scan_params(*PARAMS))

    def restated(self, d, max_nodes):
        """(scans, lengths, published) of the whole stream"""
        O = self.O
        if self.kind == "normal":
            s, l, k, _, _ = normal_restated(O, d, max_nodes)
        elif self.kind == "bytes":
            s, l, k = bytes_restated(O, self.ans, d, max_nodes, 512)
        else:
            s, l, k, _, _, _ = capsule_restated(O, self.ans, d, max_nodes)
        return s, l, k


def splits(rng, streams, n_push):
    """the streams cut into n_push pieces at different points per stream"""
    pieces = [[] for _ in range(n_push)]
    for d in streams:
        cuts = np.sort(rng.integers(0, len(d) + 1, n_push - 1))
        for t, p in enumerate(np.split(d, cuts)):
            pieces[t].append(p)
    return pieces


def cloud_rows(c, sps, n, max_scans):
    """per stream, the clouds of one cloud call: [(count, xyzi bits)]; unused slots hold count 0"""
    rows = []
    for s in range(n):
        k = min(int(sps[s]), max_scans)
        pc = c["point_counts"][s * max_scans:(s + 1) * max_scans]
        assert (pc[k:] == 0).all(), s
        rows.append([(int(pc[j]), c["xyzi"][s * max_scans + j, : pc[j]].view(np.uint32).tobytes()) for j in range(k)])
    return rows


def expected_rows(R, O, ctx, restated, kw):
    """per stream, the definition's clouds of the whole stream's scans, checked against rpl_cloud_batch_dev (flags 0
    and RPL_CLOUD_NO_FUSED) on the same scans"""
    rows, nodes, counts = [], [], []
    for scans, lens, k in restated:
        rows.append([])
        for j in range(k):
            e = O.cloud(scans[j, : lens[j]], O.cloud_params(**kw))
            rows[-1].append((e.shape[0], e.view(np.uint32).tobytes()))
        nodes.append(scans[:k])
        counts.append(lens[:k])
    nodes, counts = np.concatenate(nodes), np.concatenate(counts)
    flat = [r for row in rows for r in row]
    for flags in (0, R.CLOUD_NO_FUSED):
        for at in range(0, len(flat), ctx.max_scans):
            hi = min(at + ctx.max_scans, len(flat))
            xyzi, pc = ctx.cloud_batch(np.ascontiguousarray(nodes[at:hi]).view(R.NODE_DTYPE), counts[at:hi],
                                       R.cloud_params(flags=flags, **kw))
            got = [(int(pc[j]), xyzi[j, : pc[j]].view(np.uint32).tobytes()) for j in range(hi - at)]
            assert got == flat[at:hi], (flags, kw)
    return rows


def run(R, feed, ctx, sess, pieces, stride, settings, max_scans=MAX_SCANS):
    """pushes the pieces with host pushes; after each, one host cloud call per setting.  Returns the LaserScans per
    stream and, per setting, the clouds per stream, both concatenated over the pushes"""
    n = len(pieces[0])
    scans = [[] for _ in range(n)]
    clouds = [[[] for _ in range(n)] for _ in settings]
    for push in pieces:
        out = feed.push(sess, push, stride)
        for s, row in enumerate(_scans(out, n, max_scans)):
            scans[s] += row
        for i, prm in enumerate(settings):
            for s, row in enumerate(cloud_rows(sess.cloud(prm), out["scans_per_stream"], n, max_scans)):
                clouds[i][s] += row
    return scans, clouds


def prm_of(R, flags=0, is_new_protocol=1, **kw):
    return R.cloud_params(flags=flags, is_new_protocol=is_new_protocol, **WINDOW, **kw)


def kw_of(is_new_protocol=1, **kw):
    return dict(is_new_protocol=is_new_protocol, **WINDOW, **kw)


KINDS = [("framed", a) for a in (0x82, 0x83, 0x84, 0x86)] + [("dense", 0x85), ("normal", 0x81)] + \
        [("bytes", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("kind,ans", KINDS)
def test_pushes_give_the_whole_streams_clouds(R, oracle, kind, ans):
    """every format and session kind, each stream split into three pushes at its own points, max_nodes 8192"""
    feed = Feed(R, oracle, kind, ans)
    n, max_nodes = 8, 8192
    streams = [feed.data(s, REV_NODES[s % len(REV_NODES)] + (s // len(REV_NODES))) for s in range(n)]
    pieces = splits(np.random.default_rng(ans + len(kind)), streams, 3)
    stride = max(len(p) for push in pieces for p in push)
    ctx = R.Context(0, max_nodes, 256)
    settings = [(dict(is_new_protocol=1), 0), (dict(is_new_protocol=0, **SOR, **VOXEL), 0),
                (dict(is_new_protocol=1, **SOR, **VOXEL), R.CLOUD_NO_FUSED), (dict(is_new_protocol=0, **VOXEL), 0)]
    with feed.session(ctx, n, stride, max_nodes) as sess:
        scans, clouds = run(R, feed, ctx, sess, pieces, stride, [prm_of(R, f, **kw) for kw, f in settings])
    with feed.session(ctx, n, stride, max_nodes) as plain:  # no cloud calls in between
        plain_scans, _ = run(R, feed, ctx, plain, pieces, stride, [])
    assert scans == plain_scans
    restated = [feed.restated(d, max_nodes) for d in streams]
    lens = np.concatenate([l[:k] for _, l, k in restated])
    assert (lens > 4096).any() and (lens <= 4096).any() and (lens % 2 == 1).any()
    for i, (kw, _) in enumerate(settings):
        assert clouds[i] == expected_rows(R, oracle, ctx, restated, kw_of(**kw)), (i, kw)
    assert all(len(c) >= 2 for c in clouds[0])
    ctx.close()


@pytest.mark.parametrize("max_nodes", [4096, 8192])
def test_cloud_settings_with_duplicate_keys(R, oracle, max_nodes):
    """window only, SOR, voxel grid, both; both protocols; flags 0 and RPL_CLOUD_NO_FUSED.  HQ revolutions with
    duplicate measured keys (shared-memory kernel -> general kernel -> list-restricted post passes), odd lengths, and
    (max_nodes 8192) longer than 4096 nodes; at max_nodes 4096 the longer ones meet the holder's capacity"""
    feed = Feed(R, oracle, "framed", 0x83)
    n = 8
    streams = [hq_stream(oracle, 4, REV_NODES[s % 4] + s // 4, 700 + s, dup_share=0.002 if s % 3 else 0.0)
               for s in range(n)]
    pieces = splits(np.random.default_rng(max_nodes), streams, 2)
    stride = max(len(p) for push in pieces for p in push)
    ctx = R.Context(0, 8192, 256)
    settings = [(dict(is_new_protocol=p, **kw), f) for kw in SETTINGS for p in (0, 1) for f in (0, R.CLOUD_NO_FUSED)]
    with feed.session(ctx, n, stride, max_nodes) as sess:
        _, clouds = run(R, feed, ctx, sess, pieces, stride, [prm_of(R, f, **kw) for kw, f in settings])
    restated = [feed.restated(d, max_nodes) for d in streams]
    dup = long_dup = 0
    for scans, lens, k in restated:
        for j in range(k):
            sc = scans[j, : lens[j]]
            keys = sc["angle_z_q14"][sc["dist_mm_q2"] != 0]
            if len(np.unique(keys)) < len(keys):
                dup += 1
                long_dup += int(lens[j] > 4096)
    assert dup > 0 and (max_nodes == 4096 or long_dup > 0)
    for i, (kw, _) in enumerate(settings):
        assert clouds[i] == expected_rows(R, oracle, ctx, restated, kw_of(**kw)), (i, kw)
    ctx.close()


def dev_cloud(R, torch, sess, prm, stream=None):
    """cloud_dev into fresh device buffers on `stream` (a torch stream; None: the context's stream)"""
    ns = sess.n_streams * sess.max_scans
    xyzi = torch.full((ns, sess.max_nodes, 4), float("nan"), device="cuda")
    pc = torch.full((ns,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sess.cloud_dev(prm, xyzi.data_ptr(), pc.data_ptr(), stream=None if stream is None else stream.cuda_stream)
    return xyzi, pc


def host_of(xyzi, pc):
    import torch

    torch.cuda.synchronize()
    return {"xyzi": xyzi.cpu().numpy(), "point_counts": pc.cpu().numpy().view(np.uint32)}


def test_host_and_device_chunking_differ(R, oracle):
    """chunk_host (2 streams: large capsule strides) != chunk_dev (3 streams: the context's max_scans): a host push
    followed by cloud_dev, a push_dev followed by the host cloud"""
    import torch

    feed = Feed(R, oracle, "framed", 0x83)
    n, max_nodes, stride = 7, 8192, 8000  # 8000 HQ capsules of 781 bytes: 2 streams per 16 MiB host chunk
    streams = [hq_stream(oracle, 3, REV_NODES[s % 4] + s, 900 + s, dup_share=0.001) for s in range(n)]
    pieces = splits(np.random.default_rng(5), streams, 2)
    ctx = R.Context(0, max_nodes, 3 * MAX_SCANS)
    prms = [prm_of(R, 0, **SOR, **VOXEL), prm_of(R, R.CLOUD_NO_FUSED, **VOXEL), prm_of(R, 0)]
    got = [[[] for _ in range(n)] for _ in prms]
    with feed.session(ctx, n, stride, max_nodes) as sess:
        out = feed.push(sess, pieces[0], stride)  # host push: chunks of 2
        for i, prm in enumerate(prms):
            for s, row in enumerate(cloud_rows(host_of(*dev_cloud(R, torch, sess, prm)), out["scans_per_stream"], n,
                                               MAX_SCANS)):
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
        for i, prm in enumerate(prms):
            c = sess.cloud(prm)
            for s, row in enumerate(cloud_rows(c, sps.cpu().numpy().view(np.uint32), n, MAX_SCANS)):
                got[i][s] += row
    restated = [feed.restated(d, max_nodes) for d in streams]
    for i, kw in enumerate([kw_of(**SOR, **VOXEL), kw_of(**VOXEL), kw_of()]):
        assert got[i] == expected_rows(R, oracle, ctx, restated, kw), i
    ctx.close()


def test_side_streams_and_two_sessions(R, oracle):
    """cloud_dev on a side torch stream, then a push_dev on another stream: the clouds are the first push's.  Two
    sessions of different formats alternate on one context."""
    import torch

    n, max_nodes = 6, 8192
    feeds = [Feed(R, oracle, "framed", 0x84), Feed(R, oracle, "framed", 0x86)]
    data = [[f.data(s, REV_NODES[s % 4]) for s in range(n)] for f in feeds]
    pieces = [splits(np.random.default_rng(i), d, 2) for i, d in enumerate(data)]
    strides = [max(len(p) for push in pc for p in push) for pc in pieces]
    ctx = R.Context(0, max_nodes, 256)
    prm = prm_of(R, 0, **SOR, **VOXEL)
    side, other = torch.cuda.Stream(), torch.cuda.Stream()
    got = [[[] for _ in range(n)] for _ in feeds]
    sessions = [f.session(ctx, n, st, max_nodes) for f, st in zip(feeds, strides)]
    NS = n * MAX_SCANS
    first, dev_out = [], []
    for i, (f, sess) in enumerate(zip(feeds, sessions)):  # host push, then its clouds on the side stream
        out = f.push(sess, pieces[i][0], strides[i])
        first.append((out["scans_per_stream"].copy(), dev_cloud(R, torch, sess, prm, stream=side)))
    for i, (f, sess) in enumerate(zip(feeds, sessions)):  # the next push on another stream, before anyone waits
        buf, cnt = f.pack(pieces[i][1], strides[i])
        d_buf, d_cnt = torch.from_numpy(buf).cuda(), torch.from_numpy(cnt.view(np.int32)).cuda()
        r, it = torch.zeros((NS, max_nodes), device="cuda"), torch.zeros((NS, max_nodes), device="cuda")
        bc, inc = torch.zeros(NS, dtype=torch.int32, device="cuda"), torch.zeros(NS, device="cuda")
        sps = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.current_stream().synchronize()
        sess.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                      bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=other.cuda_stream)
        dev_out.append((d_buf, d_cnt, r, it, bc, inc, sps))
    other.synchronize()
    for i, sess in enumerate(sessions):
        sps0, (xyzi, pc) = first[i]
        for s, row in enumerate(cloud_rows(host_of(xyzi, pc), sps0, n, MAX_SCANS)):
            got[i][s] += row
        for s, row in enumerate(cloud_rows(sess.cloud(prm), dev_out[i][-1].cpu().numpy(), n, MAX_SCANS)):
            got[i][s] += row
        sess.close()
    for i, f in enumerate(feeds):
        restated = [f.restated(d, max_nodes) for d in data[i]]
        assert got[i] == expected_rows(R, oracle, ctx, restated, kw_of(**SOR, **VOXEL)), i
    ctx.close()


def test_reset_and_bad_calls(R, oracle):
    import torch

    feed = Feed(R, oracle, "framed", 0x84)
    n, max_nodes = 4, 8192
    streams = [feed.data(s, REV_NODES[s]) for s in range(n)]
    stride = max(len(d) for d in streams)
    ctx = R.Context(0, max_nodes, 64)
    prm = prm_of(R, 0, **SOR, **VOXEL)
    ns = n * MAX_SCANS
    xyzi = torch.zeros((ns, max_nodes, 4), device="cuda")
    pc = torch.zeros(ns, dtype=torch.int32, device="cuda")
    with feed.session(ctx, n, stride, max_nodes) as sess:
        for call in (lambda: sess.cloud(prm), lambda: sess.cloud_dev(prm, xyzi.data_ptr(), pc.data_ptr())):
            with pytest.raises(R.RplError) as e:  # no push yet
                call()
            assert e.value.code == R.RESULT_INVALID_DATA
        out = feed.push(sess, streams, stride)
        first = cloud_rows(sess.cloud(prm), out["scans_per_stream"], n, MAX_SCANS)
        assert sum(len(r) for r in first) >= 2 * n
        sess.reset()
        assert cloud_rows(sess.cloud(prm), out["scans_per_stream"], n, MAX_SCANS) == first
        assert cloud_rows(host_of(*dev_cloud(R, torch, sess, prm)), out["scans_per_stream"], n, MAX_SCANS) == first
        for bad in (lambda: sess.cloud(prm_of(R, 0, sor_k=33)),
                    lambda: sess.cloud(prm_of(R, 0, voxel_size=1e-7)),
                    lambda: sess.cloud_dev(prm, None, pc.data_ptr()),
                    lambda: sess.cloud_dev(prm, xyzi.data_ptr(), None)):
            with pytest.raises(R.RplError) as e:
                bad()
            assert e.value.code == R.RESULT_INVALID_DATA
        assert cloud_rows(sess.cloud(prm), out["scans_per_stream"], n, MAX_SCANS) == first  # still there
        buf, cnt = feed.pack(streams, stride)
        cnt[1] = stride + 1
        with pytest.raises(R.RplError):  # a failed push leaves no clouds to take
            sess.push(buf, cnt, R.scan_params(*PARAMS))
        with pytest.raises(R.RplError) as e:
            sess.cloud(prm)
        assert e.value.code == R.RESULT_INVALID_DATA
    ctx.close()


@pytest.mark.parametrize("mode", ["nccl", "copy"])
def test_exchange_of_a_push_at_world_1(R, oracle, mode):
    """the clouds of a push through rpl_exchange_allgather (n_scans = n_streams * max_scans, stride = max_nodes): slot 0
    holds their concatenation in slot order"""
    import torch

    feed = Feed(R, oracle, "dense", 0x85)
    n, max_nodes = 6, 8192
    streams = [feed.data(s, REV_NODES[s % 4]) for s in range(n)]
    stride = max(len(d) for d in streams)
    ctx = R.Context(0, max_nodes, 64)
    prm = prm_of(R, 0, **SOR, **VOXEL)
    with feed.session(ctx, n, stride, max_nodes) as sess:
        out = feed.push(sess, streams, stride)
        xyzi, pc = dev_cloud(R, torch, sess, prm)
        torch.cuda.synchronize()
        h = host_of(xyzi, pc)
        want = np.concatenate([h["xyzi"][j, : h["point_counts"][j]] for j in range(n * MAX_SCANS)])
        assert len(want) > 0 and sum(len(r) for r in cloud_rows(h, out["scans_per_stream"], n, MAX_SCANS)) >= 2 * n
        slot_points = len(want) + 100
        ex = R.Exchange(ctx, None, 1, 0, slot_points)
        try:
            stream = torch.cuda.current_stream().cuda_stream
            idx = ex.allgather(xyzi.data_ptr(), pc.data_ptr(), n * MAX_SCANS, max_nodes,
                               mode=R.EXCHANGE_NCCL if mode == "nccl" else R.EXCHANGE_COPY, stream=stream)
            ex.wait(idx, stream=stream)
            pts, cnt = ex.slot(idx, 0)
            count = int(dev_bytes(cnt, 4).clone().cpu().numpy().view(np.uint32)[0])
            got = dev_bytes(pts, slot_points * 16).clone().cpu().numpy().view(np.float32).reshape(-1, 4)
            ex.release(idx, stream=stream)
            ex.synchronize()
        finally:
            ex.close()
    assert count == len(want)
    assert (got[:count].view(np.uint32) == want.view(np.uint32)).all()
    ctx.close()
