"""Stamped pushes of the stream sessions (rpl_{capsule,dense,normal}_stream_push_ts*): for any split of a stream into
pushes, the scan-begin stamps published over the pushes, in order, are those of the whole stream -- the restatement's
decoder -> per-node stamps -> holder with stamps on the concatenation, each capsule (0x81: each byte) with the receive
time it was pushed with.  That restatement is pinned against the SDK's unpacker on a settable clock and its
ScanDataHolder by tests/test_stream_stamps_pieces.py.  The scans themselves are bit for bit those of the unstamped
push fed the same pieces."""
import numpy as np
import pytest

from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts, _scans
from test_gpu_dense_stream import _stream as dense_stream
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
FORMATS = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
# units (capsules; 0x81 bytes) per stream and per revolution: about 4.5 revolutions of ~2900 nodes
N_UNITS = {0x81: 5 * 14500, 0x82: 400, 0x83: 134, 0x84: 134, 0x85: 360, 0x86: 200}
PER_REV = {0x81: 5 * 2900, 0x82: 80, 0x83: 30, 0x84: 30, 0x85: 80, 0x86: 45}
MAX_NODES, MAX_SCANS = 4096, 48  # a stretch of noise bytes can open many short 0x81 scans
BIG = 10 ** 12


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _streams(O, ans, n, seed0):
    """every third stream without scan-start capsules (not 0x81 / HQ, whose scan starts are node flags)"""
    out = []
    for s in range(n):
        sync = (250 + 7 * (s % 11)) if s % 3 else None
        if ans == 0x81:
            out.append(normal_stream(N_UNITS[ans] // 5, seed0 + s, nodes_per_rev=2900, noise=50))
        elif ans == 0x85:
            out.append(dense_stream(O, N_UNITS[ans], seed0 + s, sync_every=sync))
        else:
            out.append(format_stream(O, ans, N_UNITS[ans], seed0 + s, sync_every=sync,
                                     near=(ans == 0x86 and s % 2 == 0)))
    return out


def _special_cuts(O, ans, caps, t4):
    """cuts right after and right before (the capsule holding it back) each scan-start capsule; HQ: around the capsule
    holding a scan-start node"""
    nodes, status, offs, _ = O.decode_capsules(ans, caps, int(t4[0]))
    if ans == 0x83:
        marks = sorted({int(np.searchsorted(offs, i, side="right")) - 1 for i in np.flatnonzero(nodes["flag"] & 1)})
    else:
        marks = np.flatnonzero(status & O.CAPSULE_SYNC).tolist()
    cuts = sorted({c for m in marks for c in (m, m + 1) if 0 < c < len(caps)} | {len(caps)})
    return cuts


def _restated_ts(O, ans, t4, stream, rx):
    """whole-stream scan-begin stamps: rx per capsule (0x81: per byte)"""
    if ans == 0x81:
        nodes, ends, _ = O.decode_normal(stream)
        ts = O.normal_timestamps(t4, ends, 1, rx)
        resets = None
    else:
        nodes, status, offs, _ = O.decode_capsules(ans, stream, int(t4[0]))
        ts = O.node_timestamps(ans, t4, rx, status, offs, len(nodes))
        resets = O.resets_from_capsules(status, offs)
    _, _, k, sts = O.assemble_scans_ts(nodes, ts, resets, MAX_NODES, 512)
    return sts[:k].tolist()


class Pusher:
    """one session driven by host (push_ts) or device (push_ts_dev) pushes; collects rows and stamps per stream"""

    def __init__(self, R, ctx, ans, n, stride, dev=False, dense=False):
        self.R, self.ans, self.n, self.dev = R, ans, n, dev
        if ans == 0x81:
            self.sess = R.NormalStreamSession(ctx, n, stride, MAX_NODES, MAX_SCANS)
        elif dense:
            self.sess = R.DenseStreamSession(ctx, n, stride, MAX_NODES, MAX_SCANS)
        else:
            self.sess = R.CapsuleStreamSession(ctx, ans, n, stride, MAX_NODES, MAX_SCANS)
        self.stride = stride
        self.rows, self.stamps = [[] for _ in range(n)], [[] for _ in range(n)]
        self.push_of = [[] for _ in range(n)]  # the push that published each scan
        self.t = 0

    def push(self, push, rx=None, timing=None, chunk_bytes=None):
        """push: per stream the units; rx: [n, stride] (0x81: [n, chunks]) or None for an unstamped push"""
        R, n = self.R, self.n
        if self.ans == 0x81:
            buf = np.full((n, self.stride), 0xEE, np.uint8)
        else:
            buf = np.zeros((n, self.stride, self.sess.capsule_bytes), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        kw = {}
        if rx is not None:
            kw = dict(chunk_bytes=chunk_bytes, chunk_rx_us=rx, timing=timing) if self.ans == 0x81 else \
                dict(rx_us=rx, timing=timing)
        if not self.dev:
            out = self.sess.push(buf, cnt, R.scan_params(*PARAMS), **kw)
        else:
            out = self._push_dev(buf, cnt, rx, timing, chunk_bytes)
        for s, row in enumerate(_scans(out, n, MAX_SCANS)):
            self.rows[s] += row
            k = int(out["scans_per_stream"][s])
            if rx is not None:
                st = out["scan_begin_ts_us"][s * MAX_SCANS:(s + 1) * MAX_SCANS]
                assert (st[k:] == 0).all()
                self.stamps[s] += st[:k].tolist()
            else:
                self.stamps[s] += [None] * k
            self.push_of[s] += [self.t] * k
        self.t += 1
        return out

    def _push_dev(self, buf, cnt, rx, timing, chunk_bytes):
        import torch

        dev = torch.device("cuda", 0)
        R, n, NS = self.R, self.n, self.n * MAX_SCANS
        d_buf = torch.from_numpy(buf).to(dev)
        d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
        r = torch.full((NS, MAX_NODES), -1.0, device=dev)
        it = torch.full((NS, MAX_NODES), -1.0, device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, dtype=torch.float32, device=dev)
        sps = torch.zeros(n, dtype=torch.int32, device=dev)
        ts = torch.full((NS,), -1, dtype=torch.int64, device=dev)
        args = (d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                bc.data_ptr(), inc.data_ptr(), sps.data_ptr())
        if rx is None:
            self.sess.push_dev(*args)
        else:
            d_rx = torch.from_numpy(np.ascontiguousarray(rx, np.uint64).view(np.int64)).to(dev)
            if self.ans == 0x81:
                self.sess.push_dev(*args, chunk_bytes=chunk_bytes, chunk_rx_us=d_rx.data_ptr(), timing=timing,
                                   scan_begin_ts_us=ts.data_ptr())
            else:
                self.sess.push_dev(*args, rx_us=d_rx.data_ptr(), timing=timing, scan_begin_ts_us=ts.data_ptr())
        torch.cuda.synchronize()
        return dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                    angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32),
                    scan_begin_ts_us=ts.cpu().numpy().view(np.uint64))

    def close(self):
        self.sess.close()


def _rx_times(rng, n):
    return (10_000_000 + np.cumsum(rng.integers(200, 3000, n))).astype(np.uint64)


def _capsule_rx(pieces, rx_streams, stride):
    """per push: [n, stride] receive times of the capsules each stream pushed"""
    out, at = [], [0] * len(rx_streams)
    for push in pieces:
        a = np.zeros((len(push), stride), np.uint64)
        for s, p in enumerate(push):
            a[s, : len(p)] = rx_streams[s][at[s]: at[s] + len(p)]
            at[s] += len(p)
        out.append(a)
    return out


def _normal_rx(rng, pieces, stride, chunk_bytes):
    """per push: ([n, chunks] chunk receive times) and per stream the per-byte receive times of the whole stream"""
    n = len(pieces[0])
    nch = -(-stride // chunk_bytes)
    per_push, per_byte = [], [[] for _ in range(n)]
    t = np.full(n, 10_000_000, np.uint64)
    for push in pieces:
        a = np.zeros((n, nch), np.uint64)
        for s, p in enumerate(push):
            a[s] = t[s] + np.cumsum(rng.integers(1, 500, nch)).astype(np.uint64)
            t[s] = a[s, -1]
            per_byte[s].append(np.repeat(a[s], chunk_bytes)[: len(p)])
        per_push.append(a)
    return per_push, [np.concatenate(b) if b else np.zeros(0, np.uint64) for b in per_byte]


def _cuts(O, ans, streams, t4, rng):
    rev = PER_REV[ans]
    sizes = [0, 1, 2, rev // 3, rev - 1, rev, rev + 1, 2 * rev + 2]
    cuts = [_random_cuts(rng, len(c), sizes) for c in streams]
    if ans != 0x81:
        for s in range(0, len(streams), 4):
            cuts[s] = _special_cuts(O, ans, streams[s], t4)
    return cuts


@pytest.mark.parametrize("dev", [False, True], ids=["push_ts", "push_ts_dev"])
@pytest.mark.parametrize("ans", FORMATS)
def test_random_pieces_stamp_the_whole_stream(R, oracle, ans, dev):
    O = oracle
    n = 24
    timing_t = TIMINGS[(ans + dev) % len(TIMINGS)]
    if ans != 0x83 and timing_t[0] != 31:
        timing_t = (31,) + tuple(timing_t[1:])  # the streams' revolutions are built for the 31 us jump threshold
    t4 = O.timing4(*timing_t)
    timing = R.Timing(*timing_t)
    rng = np.random.default_rng(ans * 2 + dev)
    streams = _streams(O, ans, n, 9000 + ans)
    cuts = _cuts(O, ans, streams, t4, rng)
    pieces, _ = _pieces_from_cuts(streams, cuts)
    assert any(len(p) == 0 for push in pieces[:-1] for p in push)
    stride = max(1, max(len(p) for push in pieces for p in push))
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    plain = Pusher(R, ctx, ans, n, stride)
    for push in pieces:
        plain.push(push)
    got = Pusher(R, ctx, ans, n, stride, dev=dev)
    if ans == 0x81:
        chunk_bytes = [1, 5, 64, stride][dev + 2 * (ans % 2)]
        rx_push, rx_whole = _normal_rx(rng, pieces, stride, chunk_bytes)
        for push, rx in zip(pieces, rx_push):
            got.push(push, rx, timing, chunk_bytes)
    else:
        rx_whole = [_rx_times(rng, len(c)) for c in streams]
        for push, rx in zip(pieces, _capsule_rx(pieces, rx_whole, stride)):
            got.push(push, rx, timing)
    assert got.rows == plain.rows
    n_scans = 0
    for s in range(n):
        exp = _restated_ts(O, ans, t4, streams[s], rx_whole[s])
        assert got.stamps[s] == exp, s
        n_scans += len(exp)
    assert n_scans > 2 * n
    got.close()
    plain.close()
    ctx.close()


@pytest.mark.parametrize("chunk_bytes", [1, 5, 64, "stride"])
def test_normal_chunk_sizes(R, oracle, chunk_bytes):
    """0x81 with receive times per 1, 5, 64 and >= stride_bytes bytes, on streams with inserted, dropped and flipped
    bytes and random noise"""
    O = oracle
    n = 16
    rng = np.random.default_rng(7)
    streams = _streams(O, 0x81, n, 500)
    cuts = [_random_cuts(rng, len(b), [0, 1, 4, 6, 999, 5 * 2900, 5 * 2900 + 3]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    cb = stride + 3 if chunk_bytes == "stride" else chunk_bytes
    t4 = O.timing4(*TIMINGS[1])
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    got = Pusher(R, ctx, 0x81, n, stride)
    rx_push, rx_whole = _normal_rx(rng, pieces, stride, cb)
    for push, rx in zip(pieces, rx_push):
        got.push(push, rx, R.Timing(*TIMINGS[1]), cb)
    for s in range(n):
        assert got.stamps[s] == _restated_ts(O, 0x81, t4, streams[s], rx_whole[s]), s
    got.close()
    ctx.close()


@pytest.mark.parametrize("ans", FORMATS)
def test_unstamped_push_then_stamped(R, oracle, ans):
    """unstamped pushes 0 and 2 between stamped ones: a scan published by a stamped push reports 0 when its stamp
    depends on a receive time of the last unstamped push or before it (opened before and still open across it, opened
    in it, or -- express, ultra -- released from a capsule it held), its stamp otherwise"""
    O = oracle
    n = 12
    t4 = O.timing4(*TIMINGS[0])
    timing = R.Timing(*TIMINGS[0])
    rng = np.random.default_rng(100 + ans)
    streams = _streams(O, ans, n, 9500 + ans)
    rev = PER_REV[ans]
    cuts = [[int(rng.integers(1, 2 * rev)), int(2 * rev + rng.integers(0, rev)), int(3 * rev + rng.integers(0, rev)),
             len(c)] for c in streams]
    if ans != 0x81:  # some first pushes end right after, some right before a scan-start capsule
        for s in range(0, n, 3):
            sc = _special_cuts(O, ans, streams[s], t4)
            if len(sc) > 2:
                cuts[s][0] = sc[(s // 3) % 2]
                cuts[s] = sorted(cuts[s])
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    stamped = [False, True, False, True]
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    got = Pusher(R, ctx, ans, n, stride)
    if ans == 0x81:
        rx_push, rx_whole = _normal_rx(rng, pieces, stride, 64)
    else:
        rx_whole = [_rx_times(rng, len(c)) for c in streams]
        rx_push = _capsule_rx(pieces, rx_whole, stride)
    # for each unstamped push u, the receive times of pushes 0..u moved far away: a stamp that moves with them depends
    # on what the session had before its last unstamped push
    moved = {}
    for u in (t for t in range(len(pieces)) if not stamped[t]):
        moved[u] = [r.copy() for r in rx_whole]
        for s in range(n):
            end = sum(len(pieces[t][s]) for t in range(u + 1))
            moved[u][s][:end] += np.uint64(BIG)
    for t, push in enumerate(pieces):
        if stamped[t]:
            got.push(push, rx_push[t], timing, 64)
        else:
            got.push(push)
    zeros = known = 0
    for s in range(n):
        exp = _restated_ts(O, ans, t4, streams[s], rx_whole[s])
        far = {u: _restated_ts(O, ans, t4, streams[s], m[s]) for u, m in moved.items()}
        assert len(got.stamps[s]) == len(exp)
        for j, (g, e, t) in enumerate(zip(got.stamps[s], exp, got.push_of[s])):
            if g is None:
                continue
            u = max(v for v in range(t) if not stamped[v])
            assert g == (e if e == far[u][j] else 0), (s, j)
            zeros += g == 0
            known += g != 0
    assert zeros > 0 and known > 0
    got.close()
    ctx.close()


@pytest.mark.parametrize("ans", [0x81, 0x82, 0x85])
def test_reset_mask(R, oracle, ans):
    """reset of every other stream between two pushes: those start over, stamps included"""
    O = oracle
    n = 8
    t4 = O.timing4(*TIMINGS[2])
    timing = R.Timing(*TIMINGS[2])
    rng = np.random.default_rng(ans)
    streams = _streams(O, ans, n, 9700 + ans)
    rev = PER_REV[ans]
    cuts = [[int(rev + rng.integers(0, rev)), int(2 * rev + rng.integers(0, rev)), len(c)] for c in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    if ans == 0x81:
        rx_push, rx_whole = _normal_rx(rng, pieces, stride, 5)
    else:
        rx_whole = [_rx_times(rng, len(c)) for c in streams]
        rx_push = _capsule_rx(pieces, rx_whole, stride)
    mask = np.arange(n) % 2 == 0
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    got, plain = Pusher(R, ctx, ans, n, stride), Pusher(R, ctx, ans, n, stride)
    for t, push in enumerate(pieces):
        if t == 2:
            got.sess.reset(mask)
            plain.sess.reset(mask)
        got.push(push, rx_push[t], timing, 5)
        plain.push(push)
    assert got.rows == plain.rows
    for s in range(n):
        k = cuts[s][1]
        if mask[s]:
            exp = _restated_ts(O, ans, t4, streams[s][:k], rx_whole[s][:k]) + \
                _restated_ts(O, ans, t4, streams[s][k:], rx_whole[s][k:])
        else:
            exp = _restated_ts(O, ans, t4, streams[s], rx_whole[s])
        assert got.stamps[s] == exp, s
    got.close()
    plain.close()
    ctx.close()


def test_dense_wrapper_is_the_capsule_session(R, oracle):
    O = oracle
    n = 6
    timing = R.Timing(*TIMINGS[1])
    rng = np.random.default_rng(3)
    streams = _streams(O, 0x85, n, 9900)
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, len(c), [1, 40, 79, 81, 200]) for c in streams])
    stride = max(len(p) for push in pieces for p in push)
    rx_whole = [_rx_times(rng, len(c)) for c in streams]
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    a, b = Pusher(R, ctx, 0x85, n, stride), Pusher(R, ctx, 0x85, n, stride, dense=True)
    assert isinstance(b.sess, R.DenseStreamSession)
    for push, rx in zip(pieces, _capsule_rx(pieces, rx_whole, stride)):
        a.push(push, rx, timing)
        b.push(push, rx, timing)
    assert a.rows == b.rows and a.stamps == b.stamps and sum(map(len, a.stamps)) > n
    a.close()
    b.close()
    ctx.close()


def test_argument_checks(R):
    import torch

    ctx = R.Context(0, MAX_NODES, 4 * MAX_SCANS)
    timing = R.Timing(31, 0, 0, 0)
    P = R.scan_params(*PARAMS)
    NS = 4 * MAX_SCANS
    dev = torch.device("cuda", 0)
    d = dict(r=torch.zeros((NS, MAX_NODES), device=dev), i=torch.zeros((NS, MAX_NODES), device=dev),
             b=torch.zeros(NS, dtype=torch.int32, device=dev), inc=torch.zeros(NS, device=dev),
             sps=torch.zeros(4, dtype=torch.int32, device=dev), ts=torch.zeros(NS + 1, dtype=torch.int64, device=dev),
             rx=torch.zeros(4 * 64 + 1, dtype=torch.int64, device=dev), caps=torch.zeros(4 * 10 * 84, dtype=torch.uint8,
                                                                                         device=dev),
             cnt=torch.zeros(4, dtype=torch.int32, device=dev))
    outs = (d["r"].data_ptr(), d["i"].data_ptr(), d["b"].data_ptr(), d["inc"].data_ptr(), d["sps"].data_ptr())

    def refused(fn, what):
        with pytest.raises(R.RplError) as e:
            fn()
        assert e.value.code == R.RESULT_INVALID_DATA and what in str(e.value), str(e.value)

    with R.CapsuleStreamSession(ctx, 0x82, 4, 10, MAX_NODES, MAX_SCANS) as sess:
        caps, cnt = np.zeros((4, 10, 84), np.uint8), np.zeros(4, np.uint32)
        host_out = [np.zeros(NS * MAX_NODES, np.float32), np.zeros(NS * MAX_NODES, np.float32), np.zeros(NS, np.uint32),
                    None, np.zeros(4, np.uint32), np.zeros(NS, np.uint64)]
        refused(lambda: ctx._check(sess._fn("push_ts")(
            sess._h, R.capi._p(caps), R.capi._p(cnt), None, R.capi._p(np.zeros((4, 10), np.uint64)), P,
            *[R.capi._p(a) for a in host_out])), "timing")
        base = (d["caps"].data_ptr(), d["cnt"].data_ptr(), P) + outs
        refused(lambda: sess.push_dev(*base, rx_us=None, timing=timing, scan_begin_ts_us=d["ts"].data_ptr()),
                "receive times")
        refused(lambda: sess.push_dev(*base, rx_us=d["rx"].data_ptr() + 4, timing=timing,
                                      scan_begin_ts_us=d["ts"].data_ptr()), "aligned")
        refused(lambda: sess.push_dev(*base, rx_us=d["rx"].data_ptr(), timing=timing,
                                      scan_begin_ts_us=d["ts"].data_ptr() + 4), "aligned")
        refused(lambda: sess.push_dev(*base, rx_us=d["rx"].data_ptr(), timing=None,
                                      scan_begin_ts_us=d["ts"].data_ptr()), "timing")
        refused(lambda: sess.push(caps, cnt, P, rx_us=np.zeros((4, 10), np.uint64),
                                  timing=R.Timing(0, 0, 0, 0)), "sample_duration")
        sess.push(caps, cnt, P, rx_us=np.zeros((4, 10), np.uint64), timing=timing)  # accepted
    with R.NormalStreamSession(ctx, 4, 64, MAX_NODES, MAX_SCANS) as sess:
        b, cnt = np.zeros((4, 64), np.uint8), np.zeros(4, np.uint32)
        refused(lambda: sess.push(b, cnt, P, chunk_bytes=0, chunk_rx_us=np.zeros((4, 1), np.uint64), timing=timing),
                "chunk_bytes")
        base = (d["caps"].data_ptr(), d["cnt"].data_ptr(), P) + outs
        refused(lambda: sess.push_dev(*base, chunk_bytes=1, chunk_rx_us=d["rx"].data_ptr() + 4, timing=timing,
                                      scan_begin_ts_us=d["ts"].data_ptr()), "aligned")
        refused(lambda: sess.push_dev(*base, chunk_bytes=1, chunk_rx_us=d["rx"].data_ptr(), timing=timing,
                                      scan_begin_ts_us=None), "scan_begin_ts_us")
        out = sess.push(b, cnt, P, chunk_bytes=1, chunk_rx_us=np.zeros((4, 64), np.uint64), timing=timing)
        assert (out["scan_begin_ts_us"] == 0).all()
    ctx.close()
