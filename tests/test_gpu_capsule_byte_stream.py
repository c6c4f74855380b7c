"""rpl_capsule_stream_*_bytes (CapsuleByteStreamSession): the raw serial bytes of express, HQ, ultra, dense and
ultra-dense streams, damaged and pushed in any pieces, publish exactly the scans (and stamped, the scan-begin stamps) of
the whole stream -- the SDK's unpacker and ScanDataHolder on the concatenation, as tests/test_capsule_bytes_pieces.py
pins on the CPU.  Every comparison is bit for bit on ranges, intensities, beam counts and angle increment: against one
push of the whole stream, against the restatement (framing -> oracle decoder -> holder -> ascend -> publish) and against
the framed session fed the same capsules."""
import numpy as np
import pytest

from test_capsule_bytes_pieces import FORMATS, frame_stream, raw_stream, restated, restated_scans
from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_stream import _random_cuts, _pieces_from_cuts, _scans

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
MAX_NODES, MAX_SCANS = 4096, 32


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _pack(push, stride):
    buf = np.full((len(push), stride), 0xEE, np.uint8)  # bytes past a count must not be read
    cnt = np.zeros(len(push), np.uint32)
    for s, p in enumerate(push):
        buf[s, : len(p)] = p
        cnt[s] = len(p)
    return buf, cnt


def _run(R, ctx, ans, pieces, stride, sess=None):
    """pieces: list of pushes, each a list (per stream) of byte arrays.  Returns the concatenated scans per stream and
    the state after every push."""
    n = len(pieces[0])
    own = sess is None
    sess = sess or R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, MAX_SCANS)
    got, states = [[] for _ in range(n)], []
    for push in pieces:
        buf, cnt = _pack(push, stride)
        out = sess.push(buf, cnt, R.scan_params(*PARAMS))
        for s, row in enumerate(_scans(out, n, MAX_SCANS)):
            got[s] += row
        states.append(sess.state())
    if own:
        sess.close()
    return got, states


def _oracle_rows(O, ans, b):
    e, el, ek = restated_scans(O, ans, b, MAX_NODES, 512)
    rows = []
    for k in range(ek):
        _, nodes = O.ascend(e[k, : el[k]].copy(), stable=True)
        hdr, r, it = O.publish(nodes, O.scan_params(*PARAMS, 40.0, 0.1), stable=True)
        rows.append((hdr.beam_count, r.view(np.uint32).tobytes(), it.view(np.uint32).tobytes()))
    return rows


def _check_oracle(O, ans, got, streams, which):
    for s in which:
        exp = _oracle_rows(O, ans, streams[s])
        assert len(got[s]) == len(exp), (s, len(got[s]), len(exp))
        for j, (g, e) in enumerate(zip(got[s], exp)):
            assert g[:3] == e, (s, j)


def _check_held_bytes(O, ans, states, prefixes, which):
    for t, st in enumerate(states):
        for s in which:
            assert int(st[2][s]) == frame_stream(O, ans, prefixes[t][s])[2], (t, s)


def _feature_cuts(O, ans, b):
    """byte offsets between the two sync bytes, inside a frame, inside a run of skipped bytes and right after a lone
    first-marker byte (HQ: a 0xA5 that starts no frame)"""
    cb = O.capsule_bytes(ans)
    _, last, _ = frame_stream(O, ans, b)
    starts = np.unique(last) - (cb - 1)
    covered = np.zeros(len(b), bool)
    for q in starts:
        covered[q:q + cb] = True
    skipped = np.flatnonzero(~covered)
    first = (b == 0xA5) if ans == 0x83 else ((b >> 4) == 0xA)
    lone = np.flatnonzero(first & ~covered)
    cuts = [int(q) + 1 for q in starts[::max(1, len(starts) // 8)]]
    cuts += [int(q) + cb // 2 for q in starts[1::max(1, len(starts) // 8)]]
    cuts += [int(q) for q in skipped[::max(1, len(skipped) // 12)]]
    cuts += [int(q) + 1 for q in lone[:12]]
    return sorted({c for c in cuts if 0 < c < len(b)})


@pytest.mark.parametrize("ans", FORMATS)
def test_splits_at_features(R, oracle, ans):
    """stream s split into two pushes at its own feature offset: every result equals the whole stream's"""
    b = raw_stream(oracle, ans, 700 + ans)
    cuts = _feature_cuts(oracle, ans, b)
    assert len(cuts) >= 20
    n = len(cuts)
    streams = [b] * n
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    whole, _ = _run(R, ctx, ans, [streams], len(b))
    p1, p2 = [b[:k] for k in cuts], [b[k:] for k in cuts]
    got, states = _run(R, ctx, ans, [p1, p2], len(b))
    assert got == whole
    assert len(whole[0]) >= 1
    _check_oracle(oracle, ans, got, streams, [0])
    _check_held_bytes(oracle, ans, states, [p1, streams], range(n))
    assert (states[0][2] > 0).any()
    ctx.close()


def _device_push(R, sess, buf, cnt, n, chunk_bytes=None, rx=None, timing=None):
    import torch

    dev = torch.device("cuda", 0)
    NS = n * MAX_SCANS
    d_buf = torch.from_numpy(buf).to(dev)
    d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
    r = torch.full((NS, MAX_NODES), -1.0, device=dev)
    it = torch.full((NS, MAX_NODES), -1.0, device=dev)
    bc = torch.zeros(NS, dtype=torch.int32, device=dev)
    inc = torch.zeros(NS, dtype=torch.float32, device=dev)
    sps = torch.zeros(n, dtype=torch.int32, device=dev)
    ts = torch.full((NS,), -1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    args = (d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(), bc.data_ptr(),
            inc.data_ptr(), sps.data_ptr())
    if rx is None:
        sess.push_dev(*args)
    else:
        d_rx = torch.from_numpy(np.ascontiguousarray(rx, np.uint64).view(np.int64)).to(dev)
        torch.cuda.synchronize()
        sess.push_dev(*args, chunk_bytes=chunk_bytes, chunk_rx_us=d_rx.data_ptr(), timing=timing,
                      scan_begin_ts_us=ts.data_ptr())
    sess._ctx.synchronize()
    return dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32),
                scan_begin_ts_us=ts.cpu().numpy().view(np.uint64))


def _random_pieces(O, ans, n, seed0, rng):
    cb = O.capsule_bytes(ans)
    streams = [raw_stream(O, ans, seed0 + s) for s in range(n)]
    sizes = [0, 1, 2, cb - 1, cb, cb + 1, 3 * cb + 7, 1000, 5000]
    cuts = [_random_cuts(rng, len(b), sizes) for b in streams]
    pieces, prefixes = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    return streams, pieces, prefixes, stride


@pytest.mark.parametrize("ans", FORMATS)
def test_random_pieces_host_and_device(R, oracle, ans):
    """many pushes per stream, piece sizes from 0 bytes to several frames; host pushes and push_dev agree"""
    n = 24
    rng = np.random.default_rng(ans)
    streams, pieces, prefixes, stride = _random_pieces(oracle, ans, n, 800 + ans, rng)
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    whole, _ = _run(R, ctx, ans, [streams], max(len(b) for b in streams))
    got, states = _run(R, ctx, ans, pieces, stride)
    assert got == whole
    assert sum(len(g) for g in got) >= n
    _check_oracle(oracle, ans, got, streams, range(0, n, 5))
    _check_held_bytes(oracle, ans, states[::5], prefixes[::5], range(0, n, 6))
    dgot = [[] for _ in range(n)]
    with R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, MAX_SCANS) as sess:
        for t, push in enumerate(pieces):
            buf, cnt = _pack(push, stride)
            out = _device_push(R, sess, buf, cnt, n)
            for s, row in enumerate(_scans(out, n, MAX_SCANS)):
                dgot[s] += row
            st = sess.state()
            assert all((a == b).all() for a, b in zip(st, states[t]))
    assert dgot == got
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["push_bytes_ts", "push_bytes_ts_dev"])
@pytest.mark.parametrize("ans", FORMATS)
def test_stamped_pushes_return_the_restated_stamps(R, oracle, ans, dev):
    """receive times per chunk_bytes piece of each push; a frame is stamped by the chunk holding its last byte"""
    O, n = oracle, 16
    rng = np.random.default_rng(ans * 2 + dev)
    streams, pieces, _, stride = _random_pieces(O, ans, n, 900 + ans, rng)
    t4 = O.timing4(31, 115200 * (1 + dev), 100 * dev, 0)
    timing = R.Timing(*[int(v) for v in t4])
    chunk_bytes = [1, 64, 7, stride][(ans + dev) % 4]
    nch = -(-stride // chunk_bytes)
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    plain, _ = _run(R, ctx, ans, pieces, stride)
    rows, stamps = [[] for _ in range(n)], [[] for _ in range(n)]
    per_byte = [[] for _ in range(n)]
    t_now = np.full(n, 10_000_000, np.uint64)
    with R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, MAX_SCANS) as sess:
        for push in pieces:
            rx = np.zeros((n, nch), np.uint64)
            for s, p in enumerate(push):
                rx[s] = t_now[s] + np.cumsum(rng.integers(1, 500, nch)).astype(np.uint64)
                t_now[s] = rx[s, -1]
                per_byte[s].append(np.repeat(rx[s], chunk_bytes)[: len(p)])
            buf, cnt = _pack(push, stride)
            if dev:
                out = _device_push(R, sess, buf, cnt, n, chunk_bytes, rx, timing)
            else:
                out = sess.push(buf, cnt, R.scan_params(*PARAMS), chunk_bytes=chunk_bytes, chunk_rx_us=rx, timing=timing)
            for s, row in enumerate(_scans(out, n, MAX_SCANS)):
                rows[s] += row
                k = int(out["scans_per_stream"][s])
                st = out["scan_begin_ts_us"][s * MAX_SCANS:(s + 1) * MAX_SCANS]
                assert (st[k:] == 0).all()
                stamps[s] += st[:k].tolist()
    assert rows == plain
    total = 0
    for s in range(n):
        rx_b = np.concatenate(per_byte[s])
        nodes, status, offs, last = restated(O, ans, streams[s], int(t4[0]))
        ts = O.node_timestamps(ans, t4, rx_b[last], status, offs, len(nodes))
        _, _, k, sts = O.assemble_scans_ts(nodes, ts, O.resets_from_capsules(status, offs), MAX_NODES, 512)
        assert stamps[s] == sts[:k].tolist(), s
        total += k
    assert total >= n
    ctx.close()


@pytest.mark.parametrize("ans", FORMATS)
def test_clean_bytes_equal_the_framed_session(R, oracle, ans):
    """a clean stream pushed as bytes, split at capsule boundaries, equals the framed session pushed the same capsules"""
    n, n_caps = 12, 600 if ans != 0x83 else 150
    cb = oracle.capsule_bytes(ans)
    caps = [format_stream(oracle, ans, n_caps, 1000 + s, sync_every=97 + s, bad=s % 2 == 0) for s in range(n)]
    rng = np.random.default_rng(ans)
    cuts = [_random_cuts(rng, n_caps, [0, 1, 2, 17, 60]) for _ in range(n)]
    cpieces, _ = _pieces_from_cuts(caps, cuts)
    cstride = max(1, max(len(p) for push in cpieces for p in push))
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    framed = [[] for _ in range(n)]
    with R.CapsuleStreamSession(ctx, ans, n, cstride, MAX_NODES, MAX_SCANS) as sess:
        for push in cpieces:
            buf = np.zeros((n, cstride, cb), np.uint8)
            cnt = np.zeros(n, np.uint32)
            for s, p in enumerate(push):
                buf[s, : len(p)] = p
                cnt[s] = len(p)
            for s, row in enumerate(_scans(sess.push(buf, cnt, R.scan_params(*PARAMS)), n, MAX_SCANS)):
                framed[s] += row
    bpieces = [[p.reshape(-1) for p in push] for push in cpieces]
    got, states = _run(R, ctx, ans, bpieces, cstride * cb)
    assert got == framed
    assert sum(len(g) for g in got) >= n // 2
    assert all((st[2] == 0).all() for st in states)
    ctx.close()


@pytest.mark.parametrize("ans", FORMATS)
def test_reset_mid_frame(R, oracle, ans):
    """reset while a frame is half received: a reset stream continues like a fresh session fed the rest (the handlers'
    reset() restarts the search); the others are unaffected"""
    n = 16
    cb = oracle.capsule_bytes(ans)
    streams = [raw_stream(oracle, ans, 1100 + s) for s in range(n)]
    cuts = []
    for b in streams:  # half a frame into the first frame of the second half
        starts = frame_stream(oracle, ans, b)[1] - (cb - 1)
        cuts.append(int(starts[starts >= len(b) // 2][0]) + cb // 2)
    p1, p2 = [b[:c] for b, c in zip(streams, cuts)], [b[c:] for b, c in zip(streams, cuts)]
    stride = max(len(b) for b in streams)
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    mask = np.arange(n) % 2 == 0
    with R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, MAX_SCANS) as sess:
        _run(R, ctx, ans, [p1], stride, sess=sess)
        opens0, held0, bytes0 = sess.state()
        assert (bytes0 == cb // 2).all()
        sess.reset(mask)
        opens, held, nbytes = sess.state()
        assert (opens[mask] == 0).all() and (held[mask] == 0).all() and (nbytes[mask] == 0).all()
        assert (opens[~mask] == opens0[~mask]).all() and (nbytes[~mask] == bytes0[~mask]).all()
        after, _ = _run(R, ctx, ans, [p2], stride, sess=sess)
    fresh, _ = _run(R, ctx, ans, [p2], stride)
    kept, _ = _run(R, ctx, ans, [p1, p2], stride)
    kept1, _ = _run(R, ctx, ans, [p1], stride)
    for s in range(n):
        if mask[s]:
            assert after[s] == fresh[s], s
        else:
            assert after[s] == kept[s][len(kept1[s]):], s
    ctx.close()


def test_argument_checks_capsule_and_standard_node_bytes(R, oracle):
    import ctypes as C

    L = R.lib()
    ctx = R.Context(0, MAX_NODES, 4 * MAX_SCANS)
    for ans in (0x80, 0x87):
        with pytest.raises(R.RplError) as e:
            R.CapsuleByteStreamSession(ctx, ans, 4, 1000, MAX_NODES, 8)
        assert e.value.code == R.RESULT_INVALID_DATA
    with pytest.raises(R.RplError) as e:
        R.CapsuleByteStreamSession(ctx, 0x85, 4, 0, MAX_NODES, 8)
    assert e.value.code == R.RESULT_INVALID_DATA
    out = {k: np.zeros(s, d) for k, s, d in (("r", (4 * 8, MAX_NODES), np.float32), ("b", 4 * 8, np.uint32),
                                                ("i", 4 * 8, np.float32), ("k", 4, np.uint32))}
    params = R.scan_params(*PARAMS)
    outs = [R.capi._p(out["r"]), R.capi._p(out["r"]), R.capi._p(out["b"]), R.capi._p(out["i"]), R.capi._p(out["k"])]
    raw = raw_stream(oracle, 0x85, 5)[:1000]
    buf, cnt = _pack([raw] * 4, 1000)
    with R.CapsuleByteStreamSession(ctx, 0x85, 4, 1000, MAX_NODES, 8) as bs, \
            R.CapsuleStreamSession(ctx, 0x85, 4, 12, MAX_NODES, 8) as fs:
        caps = np.zeros((4, 12, 84), np.uint8)
        ccnt = np.full(4, 12, np.uint32)
        # a framed push on a byte session, a byte push on a framed session
        assert L.rpl_capsule_stream_push(bs._h, R.capi._p(caps), R.capi._p(ccnt), 31, C.byref(params), *outs) == \
            R.RESULT_INVALID_DATA
        assert L.rpl_capsule_stream_push_bytes(fs._h, R.capi._p(buf), R.capi._p(cnt), 31, C.byref(params), *outs) == \
            R.RESULT_INVALID_DATA
        # null pointers
        assert L.rpl_capsule_stream_push_bytes(bs._h, None, R.capi._p(cnt), 31, C.byref(params), *outs) == \
            R.RESULT_INVALID_DATA
        assert L.rpl_capsule_stream_push_bytes(None, R.capi._p(buf), R.capi._p(cnt), 31, C.byref(params), *outs) == \
            R.RESULT_INVALID_DATA
        assert L.rpl_capsule_stream_create_bytes(ctx._h, 0x85, 4, 1000, MAX_NODES, 8, None) == R.RESULT_INVALID_DATA
        # a host count above the stride is refused and leaves the state alone
        with pytest.raises(R.RplError) as e:
            bs.push(buf, np.array([10, 1001, 0, 5], np.uint32), params)
        assert e.value.code == R.RESULT_INVALID_DATA and "stride" in str(e.value)
        assert all((a == 0).all() for a in bs.state())
        with pytest.raises(R.RplError) as e:
            bs.push(buf, cnt, params, chunk_bytes=0, chunk_rx_us=np.zeros((4, 1), np.uint64), timing=R.Timing(31, 0, 0, 0))
        assert e.value.code == R.RESULT_INVALID_DATA
    # on the device a count above the stride is clamped to it
    res = []
    for over in (0, 500):
        with R.CapsuleByteStreamSession(ctx, 0x85, 4, 1000, MAX_NODES, 8) as sess:
            res.append((_scans(_device_push(R, sess, buf, cnt + over, 4), 4, 8), [x.tolist() for x in sess.state()]))
    assert res[0] == res[1] and res[0][1][2] == [frame_stream(oracle, 0x85, raw)[2]] * 4
    # 0x81 standard nodes come in no capsules: a framed session of them and a framed push on their byte session are
    # refused, and state's held_bytes alone are the bytes of each stream's unfinished record
    with pytest.raises(R.RplError) as e:
        R.CapsuleStreamSession(ctx, 0x81, 4, 12, MAX_NODES, 8)
    assert e.value.code == R.RESULT_INVALID_DATA and "create_bytes" in str(e.value)
    with R.CapsuleByteStreamSession(ctx, 0x81, 4, 1000, MAX_NODES, 8) as ns:
        assert L.rpl_capsule_stream_push(ns._h, R.capi._p(caps), R.capi._p(ccnt), 31, C.byref(params), *outs) == \
            R.RESULT_INVALID_DATA
        records = np.tile(np.array([0x01, 0x01, 0, 0, 0], np.uint8), 200)  # sync bit, check bit, distance 0
        nbuf, _ = _pack([records] * 4, 1000)
        ns.push(nbuf, np.array([0, 3, 7, 12], np.uint32), params, 0)
        held = np.full(4, 99, np.uint32)
        assert L.rpl_capsule_stream_state(ns._h, None, None, R.capi._p(held)) == R.RESULT_OK
        assert held.tolist() == [0, 3, 2, 2]
    ctx.close()
