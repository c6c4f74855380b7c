"""Packed LaserScan / PointCloud2 messages of the stream sessions (rpl_*_stream_{laserscan,cloud}_msgs*): after every
push, the packed bytes are the numpy builder of tests/test_stream_msgs_pieces.py applied to that push's own outputs
(ranges, intensities, angle increments, scan-begin stamps) and the session clouds, with each scan's end stamp the
whole-stream restatement's stamp of the scan-start node that closed it."""
import numpy as np
import pytest

from oracle.cdr_oracle import parse_laserscan, parse_pointcloud2
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_stamps import _capsule_rx, _normal_rx, _rx_times, _streams
from test_normal_stream_pieces import normal_stream
from test_stream_msgs_pieces import expected_cloud, expected_laserscan, pack
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu

FORMATS = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
MAX_NODES = 4096
FRAMES = ["abcd", "laser_frame", "ab", "abc", "x" * 255, "lidar_5"]  # lengths 4, 11, 2, 3, 255, 7: residues 0..3 mod 4
OFFSET_NS = -1_234_567_891


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _restated(O, ans, t4, stream, rx):
    """whole stream: (begin, end) stamps of every published scan -- a scan [p_i, p_i+1) between two scan-start nodes is
    published iff no reset r has p_i < r <= p_i+1; its end is the stamp of node p_i+1"""
    if ans == 0x81:
        nodes, ends, _ = O.decode_normal(stream)
        ts = O.normal_timestamps(t4, ends, 1, rx)
        resets = np.zeros(0, np.int64)
    else:
        nodes, status, offs, _ = O.decode_capsules(ans, stream, int(t4[0]))
        ts = O.node_timestamps(ans, t4, rx, status, offs, len(nodes))
        resets = np.asarray(O.resets_from_capsules(status, offs), np.int64)
    p = np.flatnonzero(nodes["flag"] & 1)
    out = []
    for a, b in zip(p[:-1], p[1:]):
        if not ((resets > a) & (resets <= b)).any():
            out.append((int(ts[a]), int(ts[b])))
    _, _, k, sts = O.assemble_scans_ts(nodes, ts, None if ans == 0x81 else resets.astype(np.uint32), MAX_NODES, 4096)
    assert [b for b, _ in out] == sts[:k].tolist()
    return out


class Feed:
    """one session, host pushes; after each push the expected end stamp of every slot"""

    def __init__(self, R, O, ctx, ans, streams, pieces, t4, rng, max_scans, stamped=None):
        self.R, self.ans, self.n, self.ms = R, ans, len(streams), max_scans
        self.pieces = pieces
        self.stride = max(1, max(len(p) for push in pieces for p in push))
        if ans == 0x81:
            self.sess = R.NormalStreamSession(ctx, self.n, self.stride, MAX_NODES, max_scans)
            self.rx_push, rx_whole = _normal_rx(rng, pieces, self.stride, 64)
        else:
            self.sess = R.CapsuleStreamSession(ctx, ans, self.n, self.stride, MAX_NODES, max_scans)
            rx_whole = [_rx_times(rng, len(c)) for c in streams]
            self.rx_push = _capsule_rx(pieces, rx_whole, self.stride)
        self.whole = [_restated(O, ans, t4, s, r) for s, r in zip(streams, rx_whole)]
        self.timing = R.Timing(*TIMINGS[0])
        self.stamped = stamped or [True] * len(pieces)
        self.done = [0] * self.n  # scans published so far per stream

    def push(self, t, params):
        R, n = self.R, self.n
        push = self.pieces[t]
        if self.ans == 0x81:
            buf = np.full((n, self.stride), 0xEE, np.uint8)
        else:
            buf = np.zeros((n, self.stride, self.sess.capsule_bytes), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        if not self.stamped[t]:
            out = self.sess.push(buf, cnt, params)
            out["scan_begin_ts_us"] = np.zeros(n * self.ms, np.uint64)
        elif self.ans == 0x81:
            out = self.sess.push(buf, cnt, params, chunk_bytes=64, chunk_rx_us=self.rx_push[t], timing=self.timing)
        else:
            out = self.sess.push(buf, cnt, params, rx_us=self.rx_push[t], timing=self.timing)
        ends = np.zeros(n * self.ms, np.uint64)
        for s in range(n):
            k = int(out["scans_per_stream"][s])
            for j in range(min(k, self.ms)):
                b, e = self.whole[s][self.done[s] + j]
                if self.stamped[t]:
                    assert int(out["scan_begin_ts_us"][s * self.ms + j]) in (b, 0)
                ends[s * self.ms + j] = e if self.stamped[t] else 0
            self.done[s] += k
        out["ends"] = ends
        return out


def expected_laserscans(out, n, ms, frames, rmax, off, mode_a):
    msgs = []
    for i in range(n * ms):
        s, k = divmod(i, ms)
        m = int(out["beam_counts"][i])
        if k >= min(int(out["scans_per_stream"][s]), ms) or m == 0:
            msgs.append(None)
            continue
        b = int(out["scan_begin_ts_us"][i])
        e = int(out["ends"][i]) if b else 0
        msgs.append(expected_laserscan(frames[s], rmax[s], b, e, off, mode_a, out["ranges"][i, :m],
                                       out["intensities"][i, :m], out["angle_increment"][i]))
    return msgs


def expected_clouds(out, cloud, n, ms, frames, off):
    msgs = []
    for i in range(n * ms):
        s, k = divmod(i, ms)
        if k >= min(int(out["scans_per_stream"][s]), ms):
            msgs.append(None)
            continue
        c = int(cloud["point_counts"][i])
        msgs.append(expected_cloud(frames[s], int(out["scan_begin_ts_us"][i]), off, cloud["xyzi"][i, :c]))
    return msgs


def dev_msgs(R, sess, kind, prm, off, capacity, stream=None, guard=64):
    """the _dev form into torch buffers; returns the host view {"msgs", "msg_offsets", "msg_sizes", "total_bytes"}"""
    import torch

    dev = torch.device("cuda", 0)
    ns = sess.n_streams * sess.max_scans
    buf = torch.full((capacity + guard,), 0xA5, dtype=torch.uint8, device=dev)
    offs = torch.full((ns,), -1, dtype=torch.int64, device=dev)
    sizes = torch.full((ns,), -1, dtype=torch.int32, device=dev)
    total = torch.full((1,), -1, dtype=torch.int64, device=dev)
    fn = sess.laserscan_msgs_dev if kind == "laserscan" else sess.cloud_msgs_dev
    fn(prm, off, buf.data_ptr(), capacity, offs.data_ptr(), sizes.data_ptr(), total.data_ptr(),
       stream=None if stream is None else stream.cuda_stream)
    torch.cuda.synchronize()
    return dict(msgs=buf.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]))


def check_packed(got, exp_msgs, guard_from=None):
    offs, sizes, total = pack(exp_msgs)
    assert got["total_bytes"] == total
    assert got["msg_sizes"].tolist() == sizes.tolist()
    assert got["msg_offsets"].tolist() == offs.tolist()
    buf = got["msgs"]
    for m, o in zip(exp_msgs, offs.tolist()):
        if m is not None:
            assert bytes(buf[o: o + len(m)]) == m, o
    if guard_from is not None:
        assert (buf[total:] == guard_from).all()


def _feed(R, O, ctx, ans, n, seed, n_push=4, max_scans=48, stamped=None):
    """n streams of format ans cut at random into n_push pushes"""
    rng = np.random.default_rng(seed)
    streams = _streams(O, ans, n, 9000 + seed)
    cuts = [sorted(set(int(x) for x in rng.integers(1, len(c), n_push - 1)) | {len(c)}) for c in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    return Feed(R, O, ctx, ans, streams, pieces, O.timing4(*TIMINGS[0]), rng, max_scans, stamped)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("ans", FORMATS)
def test_every_push_packs_the_builders_messages(R, oracle, ans, dev):
    O = oracle
    n, ms = 6, 48
    ctx = R.Context(0, MAX_NODES, n * ms)
    f = _feed(R, O, ctx, ans, n, ans * 2 + dev)
    rmax = np.array([12.0, 16.0, 25.5, 8.0, 40.0, 0.5], np.float32)
    f.sess.set_frames(FRAMES, rmax)
    mode_a = dev
    prm = R.scan_params(is_new_protocol=int(ans % 2), scan_processing=int(mode_a), inverted=int(ans > 0x83),
                        apply_ascend=1)
    cprm = R.cloud_params(range_max=30.0, is_new_protocol=int(ans % 2), voxel_size=0.05 if dev else 0.0,
                          flags=R.CLOUD_NO_FUSED if ans % 2 else 0)
    n_msgs = timed = 0
    for t in range(len(f.pieces)):
        out = f.push(t, prm)
        exp = expected_laserscans(out, n, ms, FRAMES, rmax, OFFSET_NS, mode_a)
        cloud = f.sess.cloud(cprm)
        exp_c = expected_clouds(out, cloud, n, ms, FRAMES, OFFSET_NS)
        if dev:
            check_packed(dev_msgs(R, f.sess, "laserscan", prm, OFFSET_NS, 1 << 24), exp, 0xA5)
            check_packed(dev_msgs(R, f.sess, "cloud", cprm, OFFSET_NS, 1 << 25), exp_c, 0xA5)
        else:
            assert f.sess.laserscan_msgs(prm, OFFSET_NS) == exp
            assert f.sess.cloud_msgs(cprm, OFFSET_NS) == exp_c
        for m in exp:
            if m is not None:
                p = parse_laserscan(m)
                assert p["frame_id"] in FRAMES and p["scan_time"] >= 0
                n_msgs += 1
                timed += p["scan_time"] > 0 and p["sec"] > 0
        for m in exp_c:
            if m is not None:
                assert parse_pointcloud2(m)["frame_id"] in FRAMES
    assert n_msgs > n and timed > 0
    f.sess.close()
    ctx.close()


@pytest.mark.parametrize("ans", [0x81, 0x85, 0x86])
def test_overflow_and_reset_keep_the_end_stamp(R, oracle, ans):
    """max_scans 1: the stored slot's end is the begin of the first dropped scan; a reset after the push changes nothing
    about its messages"""
    O = oracle
    n, ms = 4, 1
    ctx = R.Context(0, MAX_NODES, n * ms)
    f = _feed(R, O, ctx, ans, n, 77 + ans, n_push=2, max_scans=ms)
    prm = R.scan_params(1, 0, 0, 1)
    checked = 0
    for t in range(len(f.pieces)):
        out = f.push(t, prm)
        exp = expected_laserscans(out, n, ms, ["laser_frame"] * n, [12.0] * n, 0, False)
        got = f.sess.laserscan_msgs(prm)
        assert got == exp
        if t == len(f.pieces) - 1:  # a reset after the last push
            f.sess.reset()
            assert f.sess.laserscan_msgs(prm) == exp
        for s in range(n):
            if int(out["scans_per_stream"][s]) > 1 and exp[s] is not None:
                p = parse_laserscan(exp[s])
                b, e = f.whole[s][f.done[s] - int(out["scans_per_stream"][s])]
                assert p["scan_time"] == np.float32(max(e - b, 0) * 1000 / 1e9)
                checked += e > b  # 0x81 noise opens short scans inside one receive chunk: e == b, period 0
    assert checked > 0
    f.sess.close()
    ctx.close()


@pytest.mark.parametrize("ans", [0x82, 0x85])
def test_byte_session(R, oracle, ans):
    O = oracle
    n, ms = 4, 48
    ctx = R.Context(0, MAX_NODES, n * ms)
    rng = np.random.default_rng(ans)
    streams = [c.reshape(-1) for c in _streams(O, ans, n, 4000 + ans)]
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    sess = R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, ms)
    rx_push, _ = _normal_rx(rng, pieces, stride, 64)
    prm = R.scan_params(0, 1, 1, 1)
    cprm = R.cloud_params()
    timing = R.Timing(*TIMINGS[0])
    seen = 0
    for t, push in enumerate(pieces):
        buf = np.zeros((n, stride), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        out = sess.push(buf, cnt, prm, chunk_bytes=64, chunk_rx_us=rx_push[t], timing=timing)
        got = sess.laserscan_msgs(prm, 5)
        for i, m in enumerate(got):
            s, k = divmod(i, ms)
            bc = int(out["beam_counts"][i])
            assert (m is None) == (k >= min(int(out["scans_per_stream"][s]), ms) or bc == 0)
            if m is None:
                continue
            p = parse_laserscan(m)
            assert p["ranges"].tobytes() == out["ranges"][i, :bc].tobytes()
            assert (p["sec"], p["nanosec"]) == divmod(int(out["scan_begin_ts_us"][i]) * 1000 + 5, 10 ** 9)
            seen += 1
        assert len(sess.cloud_msgs(cprm)) == n * ms
    assert seen > n
    sess.close()
    ctx.close()


def test_unstamped_and_mixed_pushes(R, oracle):
    """an unstamped push's messages carry stamp {0, 0} and no period; a stamped push after it its own begin stamps"""
    O = oracle
    n, ms = 6, 48
    ctx = R.Context(0, MAX_NODES, n * ms)
    f = _feed(R, O, ctx, 0x84, n, 5, n_push=4, stamped=[False, True, False, True])
    prm = R.scan_params(1, 0, 0, 1)
    for t in range(len(f.pieces)):
        out = f.push(t, prm)
        got = f.sess.laserscan_msgs(prm, 10 ** 9)
        for i, m in enumerate(got):
            if m is None:
                continue
            p = parse_laserscan(m)
            b = int(out["scan_begin_ts_us"][i])
            if not f.stamped[t]:
                assert (p["sec"], p["nanosec"], p["scan_time"], p["time_increment"]) == (0, 0, 0, 0)
            else:
                assert (p["sec"], p["nanosec"]) == ((divmod(b * 1000 + 10 ** 9, 10 ** 9)) if b else (0, 0))
    f.sess.close()
    ctx.close()


def test_unmeasured_scans_capacity_and_side_streams(R, oracle):
    """all-unmeasured revolutions: no LaserScan, an empty cloud message; capacity one byte short writes nothing and
    reports the total; device calls on a side stream order against the pushes"""
    import torch

    O = oracle
    n, ms = 3, 48
    streams = [normal_stream(2900 * 3, 31 + s, nodes_per_rev=2900, noise=0) for s in range(n)]
    # stream 1: every distance zeroed (the last two bytes of each record) -> unmeasured revolutions
    b = streams[1].copy()
    _, ends, _ = O.decode_normal(b)
    ends = np.asarray(ends, np.int64)
    b[ends] = 0
    b[ends - 1] = 0
    streams[1] = b
    ctx = R.Context(0, MAX_NODES, n * ms)
    stride = max(len(x) for x in streams)
    sess = R.NormalStreamSession(ctx, n, stride, MAX_NODES, ms)
    buf = np.zeros((n, stride), np.uint8)
    for s, x in enumerate(streams):
        buf[s, : len(x)] = x
    prm = R.scan_params(0, 0, 0, 1)
    out = sess.push(buf, np.array([len(x) for x in streams], np.uint32), prm)
    ls = sess.laserscan_msgs(prm)
    cl = sess.cloud_msgs(R.cloud_params())
    k1 = int(out["scans_per_stream"][1])
    assert k1 > 0 and all(ls[ms + j] is None for j in range(ms))
    assert all(parse_pointcloud2(cl[ms + j])["width"] == 0 for j in range(k1))
    # capacity: exactly the total fits, one byte short writes nothing
    full = sess.laserscan_msgs(prm, packed=True)
    total = full["total_bytes"]
    fit = sess.laserscan_msgs(prm, msgs=np.full(total, 0x5A, np.uint8), packed=True)
    assert fit["result"] == 0 and bytes(fit["msgs"]) == bytes(full["msgs"][:total])
    short = sess.laserscan_msgs(prm, msgs=np.full(total - 1, 0x5A, np.uint8), packed=True)
    assert short["result"] == R.capi.RESULT_INSUFFICIENT_MEMORY and short["total_bytes"] == total
    assert (short["msg_sizes"] == 0).all() and (short["msgs"] == 0x5A).all()
    d = dev_msgs(R, sess, "laserscan", prm, 0, total - 1, guard=32)
    assert d["total_bytes"] == total and (d["msg_sizes"] == 0).all() and (d["msgs"] == 0xA5).all()
    # side stream: a device push of the same bytes on a fresh session, messages on another stream
    sess2 = R.NormalStreamSession(ctx, n, stride, MAX_NODES, ms)
    dev = torch.device("cuda", 0)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    NS = n * ms
    with torch.cuda.stream(s1):
        d_buf = torch.from_numpy(buf).to(dev)
        d_cnt = torch.tensor([len(x) for x in streams], dtype=torch.int32, device=dev)
        r = torch.zeros((NS, MAX_NODES), device=dev)
        it = torch.zeros((NS, MAX_NODES), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n, dtype=torch.int32, device=dev)
    sess2.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                   inc.data_ptr(), sps.data_ptr(), stream=s1.cuda_stream)
    got = dev_msgs(R, sess2, "laserscan", prm, 0, 1 << 22, stream=s2)
    check_packed(got, [m for m in ls])
    sess2.close()
    sess.close()
    ctx.close()


def test_argument_checks(R, oracle):
    ctx = R.Context(0, MAX_NODES, 4 * 48)
    prm, cprm = R.scan_params(), R.cloud_params()

    def refused(fn, what, code=None):
        with pytest.raises(R.RplError) as e:
            fn()
        assert e.value.code == (code or R.RESULT_INVALID_DATA) and what in str(e.value), str(e.value)

    with R.CapsuleStreamSession(ctx, 0x82, 4, 10, MAX_NODES, 48) as sess:
        refused(lambda: sess.laserscan_msgs(prm), "no messages")
        refused(lambda: sess.cloud_msgs(cprm), "no messages")
        refused(lambda: sess.set_frames(["a", "b", "c", "x" * 256]), "255")
        ns = 4 * 48
        z = np.zeros(ns, np.uint64)
        refused(lambda: ctx._check(sess._fn("laserscan_msgs")(sess._h, prm, 0, None, 0, R.capi._p(z),
                                                              R.capi._p(z), R.capi._p(z))), "null")
        sess.push(np.zeros((4, 10, 84), np.uint8), np.zeros(4, np.uint32), prm)
        assert sess.laserscan_msgs(prm) == [None] * ns
        assert sess.cloud_msgs(cprm) == [None] * ns
        refused(lambda: sess.cloud_msgs(R.cloud_params(sor_k=33)), "sor_k")
        refused(lambda: sess.laserscan_msgs_dev(prm, 0, 8, 100, 16, 16, 16), "aligned")
        refused(lambda: ctx._check(sess._fn("laserscan_msgs")(sess._h, None, 0, R.capi._p(z), 8, R.capi._p(z),
                                                              R.capi._p(z), R.capi._p(z))), "null")
        sess.set_frames(["a", "b", "c", "d"])  # range_max kept
    ctx.close()
