"""Stream sessions whose pushes run in several chunks, and pushes that run past a session's lists and scan slots.

Chunks: 8 streams on a context whose max_scans is 3 x the session's, so that a device push runs in chunks of 3, 3 and
2 streams and a host push keeps both lanes in flight; each stream is split into random pieces of its own.  Stamped
framed and 0x81 pushes and byte pushes (host and device, unstamped and stamped) give the whole stream's scans, stamps
and state; after a multi-chunk byte push the session clouds equal rpl_cloud_batch on the same scans.

Past the lists and slots: a push that brings more than 4096 scan starts per stream (0x81 revolutions of 2-5 records),
more than 1024 scan-reset requests (express and dense scan-start capsules every 1-2 capsules), or, dense, more scan
starts than the decoder lists (2 * max_scans + 64), each with a revolution carried in from the push before.  Two
sessions take the same pieces: one with max_scans large enough to store every scan, which equals the whole stream's
restatement, and one with max_scans 4, which publishes as many scans, stores the first 4 of them (rows, stamps,
clouds) and carries on exactly as the large one."""
import numpy as np
import pytest

from test_capsule_oracle_vs_ref import make_capsules
from test_capsule_stream_pieces import restated_scans as capsule_restated
from test_decode_oracle_vs_ref import make_stream
from test_gpu_capsule_byte_stream import _device_push, _pack, _random_pieces
from test_gpu_capsule_byte_stream import MAX_SCANS as BYTE_SCANS
from test_gpu_capsule_stream import _pieces_from_cuts, _scans
from test_gpu_stream_cloud import Feed, cloud_rows, dev_cloud, expected_rows, host_of, kw_of, prm_of
from test_gpu_stream_stamps import MAX_NODES as STAMP_NODES, MAX_SCANS as STAMP_SCANS
from test_gpu_stream_stamps import Pusher, _capsule_rx, _cuts, _normal_rx, _restated_ts, _rx_times, _streams
from test_normal_stream_pieces import normal_stream, restated_scans as normal_restated
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
N = 8  # streams: device chunks of 3, 3 and 2


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


# ---- B. sessions across chunks and lanes -----------------------------------------------------------------------------
def _stamped_run(R, O, ctx, ans, streams, pieces, stride, dev, rng, timing, t4):
    got = Pusher(R, ctx, ans, N, stride, dev=dev)
    if ans == 0x81:
        rx_push, rx_whole = _normal_rx(rng, pieces, stride, 64)
        for push, rx in zip(pieces, rx_push):
            got.push(push, rx, timing, 64)
    else:
        rx_whole = [_rx_times(rng, len(c)) for c in streams]
        for push, rx in zip(pieces, _capsule_rx(pieces, rx_whole, stride)):
            got.push(push, rx, timing)
    return got, rx_whole


@pytest.mark.parametrize("dev", [False, True], ids=["push_ts", "push_ts_dev"])
@pytest.mark.parametrize("ans", [0x81, 0x82, 0x83, 0x84, 0x85, 0x86])
def test_stamped_pushes_across_chunks(R, oracle, ans, dev):
    O = oracle
    t4 = O.timing4(*TIMINGS[0])
    timing = R.Timing(*TIMINGS[0])
    rng = np.random.default_rng(300 + 2 * ans + dev)
    streams = _streams(O, ans, N, 12000 + ans)
    pieces, _ = _pieces_from_cuts(streams, _cuts(O, ans, streams, t4, rng))
    stride = max(1, max(len(p) for push in pieces for p in push))
    ctx = R.Context(0, STAMP_NODES, 3 * STAMP_SCANS)
    whole = Pusher(R, ctx, ans, N, max(len(c) for c in streams))
    whole.push(streams)
    got, rx_whole = _stamped_run(R, O, ctx, ans, streams, pieces, stride, dev, rng, timing, t4)
    assert got.rows == whole.rows
    assert sum(len(r) for r in got.rows) > 2 * N
    for s in range(N):
        assert got.stamps[s] == _restated_ts(O, ans, t4, streams[s], rx_whole[s]), s
    assert all((a == b).all() for a, b in zip(got.sess.state(), whole.sess.state()))
    got.close()
    whole.close()
    ctx.close()


@pytest.mark.parametrize("stamped", [False, True], ids=["unstamped", "stamped"])
@pytest.mark.parametrize("dev", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("ans", [0x82, 0x83, 0x84, 0x85, 0x86])
def test_byte_pushes_across_chunks(R, oracle, ans, dev, stamped):
    O = oracle
    rng = np.random.default_rng(ans * 4 + 2 * dev + stamped)
    streams, pieces, _, stride = _random_pieces(O, ans, N, 1300 + ans, rng)
    t4 = O.timing4(31, 115200, 0, 0)
    timing = R.Timing(*[int(v) for v in t4])
    chunk_bytes = 64
    nch = -(-stride // chunk_bytes)
    ctx = R.Context(0, 4096, 3 * BYTE_SCANS)
    wstride = max(len(b) for b in streams)
    with R.CapsuleByteStreamSession(ctx, ans, N, wstride, 4096, BYTE_SCANS) as whole:
        buf, cnt = _pack(streams, wstride)
        want = _scans(whole.push(buf, cnt, R.scan_params(*PARAMS)), N, BYTE_SCANS)
        want_state = whole.state()
    rows, stamps, per_byte = [[] for _ in range(N)], [[] for _ in range(N)], [[] for _ in range(N)]
    t_now = np.full(N, 10_000_000, np.uint64)
    with R.CapsuleByteStreamSession(ctx, ans, N, stride, 4096, BYTE_SCANS) as sess:
        for push in pieces:
            buf, cnt = _pack(push, stride)
            kw = {}
            if stamped:
                rx = np.zeros((N, nch), np.uint64)
                for s, p in enumerate(push):
                    rx[s] = t_now[s] + np.cumsum(rng.integers(1, 500, nch)).astype(np.uint64)
                    t_now[s] = rx[s, -1]
                    per_byte[s].append(np.repeat(rx[s], chunk_bytes)[: len(p)])
                kw = dict(chunk_bytes=chunk_bytes, rx=rx, timing=timing)
            if dev:
                out = _device_push(R, sess, buf, cnt, N, **kw)
            elif stamped:
                out = sess.push(buf, cnt, R.scan_params(*PARAMS), chunk_bytes=chunk_bytes, chunk_rx_us=kw["rx"],
                                timing=timing)
            else:
                out = sess.push(buf, cnt, R.scan_params(*PARAMS))
            for s, row in enumerate(_scans(out, N, BYTE_SCANS)):
                rows[s] += row
                if stamped:
                    stamps[s] += out["scan_begin_ts_us"][s * BYTE_SCANS: s * BYTE_SCANS + len(row)].tolist()
        assert all((a == b).all() for a, b in zip(sess.state(), want_state))
    assert rows == want
    assert sum(len(r) for r in rows) >= N
    if stamped:
        from test_capsule_bytes_pieces import restated

        for s in range(N):
            nodes, status, offs, last = restated(O, ans, streams[s], int(t4[0]))
            ts = O.node_timestamps(ans, t4, np.concatenate(per_byte[s])[last], status, offs, len(nodes))
            _, _, k, sts = O.assemble_scans_ts(nodes, ts, O.resets_from_capsules(status, offs), 4096, 512)
            assert stamps[s] == sts[:k].tolist(), s
    ctx.close()


@pytest.mark.parametrize("stride,max_scans", [(None, 3), (8000, 3)], ids=["chunks-of-3", "host-chunks-of-2"])
def test_byte_session_clouds_across_chunks(R, oracle, stride, max_scans):
    """clouds after multi-chunk byte pushes (host and device), host and device cloud calls; with 8000-capsule strides
    of HQ bytes the host pushes run 2 streams per chunk and the device pushes 3"""
    import torch

    feed = Feed(R, oracle, "bytes", 0x83 if stride else 0x84)
    max_nodes, slots = 8192, 24
    streams = [feed.data(s, (2950, 5801, 4097)[s % 3]) for s in range(N)]
    rng = np.random.default_rng(17)
    pieces = [[] for _ in range(3)]
    for d in streams:
        for t, p in enumerate(np.split(d, np.sort(rng.integers(0, len(d) + 1, 2)))):
            pieces[t].append(p)
    stride = stride * 781 if stride else max(len(p) for push in pieces for p in push)
    ctx = R.Context(0, max_nodes, max_scans * slots)
    prm, kw = prm_of(R, 0, sor_k=8, sor_alpha=1.0, voxel_size=0.05), kw_of(sor_k=8, sor_alpha=1.0, voxel_size=0.05)
    host_rows, dev_rows = [[] for _ in range(N)], [[] for _ in range(N)]
    NS = N * slots
    with feed.session(ctx, N, stride, max_nodes, slots) as sess:
        for t, push in enumerate(pieces):
            buf, cnt = feed.pack(push, stride)
            if t % 2 == 0:
                sps = sess.push(buf, cnt, R.scan_params(*PARAMS))["scans_per_stream"]
            else:
                d_buf, d_cnt = torch.from_numpy(buf).cuda(), torch.from_numpy(cnt.view(np.int32)).cuda()
                r, it = torch.zeros((NS, max_nodes), device="cuda"), torch.zeros((NS, max_nodes), device="cuda")
                bc, inc = torch.zeros(NS, dtype=torch.int32, device="cuda"), torch.zeros(NS, device="cuda")
                d_sps = torch.zeros(N, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                sess.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                              bc.data_ptr(), inc.data_ptr(), d_sps.data_ptr())
                ctx.synchronize()
                sps = d_sps.cpu().numpy().view(np.uint32)
            for s, row in enumerate(cloud_rows(sess.cloud(prm), sps, N, slots)):
                host_rows[s] += row
            for s, row in enumerate(cloud_rows(host_of(*dev_cloud(R, torch, sess, prm)), sps, N, slots)):
                dev_rows[s] += row
    restated = [feed.restated(d, max_nodes) for d in streams]
    want = expected_rows(R, oracle, ctx, restated, kw)
    assert host_rows == want and dev_rows == want
    assert all(len(r) >= 2 for r in want)
    ctx.close()


# ---- C. pushes past the session's lists and slots --------------------------------------------------------------------
SMALL_NODES = 64
TIMING = TIMINGS[0]


def _case(O, kind, s):
    """(answer type, the stream, its pieces): a short first push that leaves a revolution open, the bulk push, a
    last push of a few scans"""
    if kind == "normal":  # revolutions of 2-5 records: more than 4096 scan starts in the bulk push
        rev = 2 + s % 4
        d = normal_stream(4400 * rev, 40 + s, nodes_per_rev=rev, bad=False, noise=0)
        cut0, cut1 = 5 * (3 * rev + 1) + 2, len(d) - 5 * 3 * rev
        return 0x81, d, [d[:cut0], d[cut0:cut1], d[cut1:]]
    if kind == "dense-list":  # scan starts past the decoder's list of the small session (72), below 4096
        d = make_stream(O, 1800, 10.0, seed=50 + s)
        return 0x85, d, [d[:15], d[15:1790], d[1790:]]
    ans = 0x85 if kind == "dense-resets" else 0x82
    gen = (lambda n, cpr, seed, se=None: make_stream(O, n, cpr, seed=seed, sync_every=se)) if ans == 0x85 else \
        (lambda n, cpr, seed, se=None: make_capsules(O, ans, n, cpr, seed=seed, sync_every=se))
    # scans, a run of scan-start capsules every 1-2 capsules (more than 1024 reset requests), scans again
    d = np.concatenate([gen(300, 10.0, 60 + s), gen(2300, 10.0, 70 + s, 1 + s % 2), gen(600, 10.0, 80 + s)])
    return ans, d, [d[:155], d[155:len(d) - 15], d[len(d) - 15:]]


def _session(R, ctx, ans, n, stride, max_scans):
    if ans == 0x81:
        return R.NormalStreamSession(ctx, n, stride, SMALL_NODES, max_scans)
    if ans == 0x85:
        return R.DenseStreamSession(ctx, n, stride, SMALL_NODES, max_scans)
    return R.CapsuleStreamSession(ctx, ans, n, stride, SMALL_NODES, max_scans)


def _push(R, sess, ans, push, stride, rx_at):
    """one stamped host push; rx_at: per stream the receive time of its first unit in this push"""
    n = len(push)
    if ans == 0x81:
        buf = np.zeros((n, stride), np.uint8)
        nch = -(-stride // 64)
        rx = np.array([rx_at[s] + 7 * np.arange(nch) for s in range(n)], np.uint64)
    else:
        buf = np.zeros((n, stride, push[0].shape[1]), np.uint8)
        rx = np.array([rx_at[s] + 300 * np.arange(stride) for s in range(n)], np.uint64)
    cnt = np.zeros(n, np.uint32)
    for s, p in enumerate(push):
        buf[s, : len(p)] = p
        cnt[s] = len(p)
    if ans == 0x81:
        return sess.push(buf, cnt, R.scan_params(*PARAMS), chunk_bytes=64, chunk_rx_us=rx, timing=R.Timing(*TIMING))
    return sess.push(buf, cnt, R.scan_params(*PARAMS), rx_us=rx, timing=R.Timing(*TIMING))


@pytest.mark.parametrize("kind", ["normal", "express-resets", "dense-resets", "dense-list"])
def test_pushes_past_lists_and_slots(R, oracle, kind):
    O = oracle
    n = 3
    cases = [_case(O, kind, s) for s in range(n)]
    ans = cases[0][0]
    pieces = [[c[2][t] for c in cases] for t in range(3)]
    stride = max(len(p) for push in pieces for p in push)
    # the whole stream's scans (and how many of them the bulk push closes)
    restated = []
    for _, d, _ in cases:
        if ans == 0x81:
            sc, ln, k, _, _ = normal_restated(O, d, SMALL_NODES, 20000)
        else:
            sc, ln, k, nodes, status, offs = capsule_restated(O, ans, d, SMALL_NODES, 20000)
            if kind != "dense-list":
                assert len(O.resets_from_capsules(status, offs)) > 1024
        restated.append((sc, ln, k))
    big_scans = max(k for _, _, k in restated) + 8
    if kind == "dense-list":
        assert all(k > 2 * 4 + 64 for _, _, k in restated) and big_scans < 4096
    ctx = R.Context(0, SMALL_NODES, n * big_scans)
    big, small = _session(R, ctx, ans, n, stride, big_scans), _session(R, ctx, ans, n, stride, 4)
    rx_at = np.full(n, 10_000_000, np.uint64)
    prm = R.cloud_params(is_new_protocol=1, range_min=0.15, range_max=40.0)
    big_rows = [[] for _ in range(n)]
    for t, push in enumerate(pieces):
        ob, os_ = _push(R, big, ans, push, stride, rx_at), _push(R, small, ans, push, stride, rx_at)
        rx_at += np.uint64(10_000_000)
        k = ob["scans_per_stream"]
        assert (os_["scans_per_stream"] == k).all(), t
        rb = _scans(ob, n, big_scans)
        for s in range(n):
            big_rows[s] += rb[s]
        if t == 1:
            assert (k > 4).all() and (k > (4096 if kind == "normal" else 0)).all()
        # the small session's 4 slots: the large one's first 4 scans, their stamps and clouds
        ks = np.minimum(k, 4)
        cut = dict(os_)
        cut["scans_per_stream"] = ks
        assert _scans(cut, n, 4) == [r[:4] for r in rb], t
        for s in range(n):
            assert (os_["scan_begin_ts_us"][4 * s: 4 * s + ks[s]] ==
                    ob["scan_begin_ts_us"][big_scans * s: big_scans * s + ks[s]]).all(), (t, s)
        cb = [r[:4] for r in cloud_rows(big.cloud(prm), k, n, big_scans)]
        cs = cloud_rows(small.cloud(prm), k, n, 4)
        assert cb == cs, t
        assert all((a == b).all() for a, b in zip(big.state(), small.state())), t
    # the large session holds the whole stream's scans
    for s, (sc, ln, k) in enumerate(restated):
        assert len(big_rows[s]) == k, s
        for j in range(0, k, max(1, k // 200)):  # a sample of the scans through the oracle
            _, nodes = O.ascend(sc[j, : ln[j]].copy(), stable=True)
            hdr, r, it = O.publish(nodes, O.scan_params(*PARAMS, 40.0, 0.1), stable=True)
            assert big_rows[s][j][:3] == (hdr.beam_count, r.view(np.uint32).tobytes(), it.view(np.uint32).tobytes()), \
                (s, j)
    big.close()
    small.close()
    ctx.close()
