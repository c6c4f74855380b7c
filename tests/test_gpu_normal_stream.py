"""The standard-node session (NormalStreamSession, rpl_capsule_stream_*_bytes on 0x81): a raw 0x81 standard-node byte
stream pushed in pieces publishes exactly the scans of the whole stream -- the SDK's UnpackerHandler_NormalNode ->
ScanDataHolder -> ascendScanData -> publish_scan on the concatenation (pinned on the CPU by
tests/test_normal_stream_pieces.py).  Every comparison is bit for bit on ranges, intensities, beam counts and angle
increment: against one push of the whole stream, against the restatement (oracle decode_normal -> assemble_scans ->
ascend -> publish, stable tie rule) and, where oracle/_ref is built, the SDK's own decoder and holder."""
import numpy as np
import pytest

from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts, _scans
from test_normal_stream_pieces import NODES_PER_REV, normal_stream, restated_scans

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend


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


def _run(R, ctx, pieces, max_nodes, max_scans, params=PARAMS, sess=None, stride=None):
    """pieces: list of pushes, each a list (per stream) of byte arrays.  Returns the concatenated scans per stream and
    the state after every push."""
    n = len(pieces[0])
    stride = stride or max(1, max(len(p) for push in pieces for p in push))
    own = sess is None
    sess = sess or R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans)
    got, states = [[] for _ in range(n)], []
    for push in pieces:
        buf, cnt = _pack(push, sess.stride_bytes)
        out = sess.push(buf, cnt, R.scan_params(*params))
        for s, row in enumerate(_scans(out, n, max_scans)):
            got[s] += row
        states.append(sess.state())
    if own:
        sess.close()
    return got, states


def _oracle_rows(O, b, max_nodes, params=PARAMS):
    e, el, ek, _, _ = restated_scans(O, b, max_nodes)
    rows = []
    for k in range(ek):
        nodes = e[k, : el[k]].copy()
        if params[3]:
            _, nodes = O.ascend(nodes, stable=True)
        hdr, r, it = O.publish(nodes, O.scan_params(params[0], params[1], params[2], params[3], 40.0, 0.1), stable=True)
        rows.append((hdr.beam_count, r.view(np.uint32).tobytes(), it.view(np.uint32).tobytes()))
    return rows


def _expected_state(O, b, max_nodes):
    """(open nodes, held bytes) after the bytes b: the holder's scan in progress (nodes since the last scan start,
    capped), and the byte machine's state"""
    nodes, _, pos = O.decode_normal(b)
    starts = np.nonzero(nodes["flag"] & 1)[0]
    if len(starts) == 0:
        return 0, pos
    return min(len(nodes) - int(starts[-1]), max_nodes), pos


def _check_states(O, states, prefixes, max_nodes, which):
    """states[t] after push t against the restatement on prefixes[t][s] (the bytes pushed so far)"""
    for t, st in enumerate(states):
        for s in which:
            assert (int(st[0][s]), int(st[1][s])) == _expected_state(O, prefixes[t][s], max_nodes), (t, s)


def _check_oracle(O, got, streams, max_nodes, which, params=PARAMS):
    for s in which:
        exp = _oracle_rows(O, streams[s], max_nodes, params)
        assert len(got[s]) == len(exp), (s, len(got[s]), len(exp))
        for j, (g, e) in enumerate(zip(got[s], exp)):
            assert g[:3] == e, (s, j)


def _check_ref(O, streams, max_nodes, which):
    """where oracle/_ref is built: the SDK's own decoder and holder give the restatement's scans on these streams"""
    if not (O.have_ref() and O.have_ref_holder()):
        return
    for s in which:
        rn, _ = O.ref_unpack(0x81, streams[s], 31, 0)
        rs, rl, rk = O.ref_assemble_scans(rn, None, max_nodes, 512)
        e, el, ek, _, _ = restated_scans(O, streams[s], max_nodes)
        assert rk == ek and (rl == el).all(), s
        for k in range(min(ek, 512)):
            assert (rs[k, : rl[k]].view(np.uint64) == e[k, : el[k]].view(np.uint64)).all(), (s, k)


def _featured_stream(n_records=4 * NODES_PER_REV + 100, seed=41):
    """a clean stream with, at known byte positions: its first scan-start record, a record whose check bit fails, a
    dropped byte (the machine resynchronises over the records after it), 7 inserted noise bytes, and the last record
    of the first full revolution.  Returns (bytes, {feature: byte position})."""
    b = normal_stream(n_records, seed, bad=False).copy()
    r0 = int(np.nonzero(b[0::5] & 1)[0][0])
    r_chk, r_del, r_ins, r_last = r0 + 500, r0 + 1000, r0 + 1500, r0 + NODES_PER_REV - 1
    b[5 * r_chk + 1] &= 0xFE
    noise = np.random.default_rng(seed).integers(0, 256, 7, dtype=np.uint8)
    b = np.concatenate([b[: 5 * r_ins], noise, b[5 * r_ins:]])
    b = np.delete(b, 5 * r_del + 2)
    feats = {"start": 5 * r0, "check": 5 * r_chk + 1, "resync": 5 * r_del + 2, "noise": 5 * r_ins - 1 + 3,
             "last": 5 * r_last - 1 + 7 + 5}
    return b, feats


def test_every_split_around_features(R, oracle):
    """each stream is split into two pushes at one byte offset, in windows around a scan-start record, a record whose
    check bit fails, a resynchronisation in progress, noise, and a revolution's last record"""
    b, feats = _featured_stream()
    cuts = [f + d for f in feats.values() for d in range(-7, 8)] + list(range(feats["resync"] + 8, feats["resync"] + 40))
    n, max_nodes, max_scans = len(cuts), 4096, 16
    streams = [b] * n
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], max_nodes, max_scans)
    p1, p2 = [b[:k] for k in cuts], [b[k:] for k in cuts]
    got, states = _run(R, ctx, [p1, p2], max_nodes, max_scans, stride=len(b))
    assert got == whole
    assert len(whole[0]) >= 3
    _check_oracle(oracle, got, streams, max_nodes, [0])
    _check_ref(oracle, streams, max_nodes, [0])
    _check_states(oracle, states, [p1, streams], max_nodes, range(n))
    held = states[0][1]
    assert set(int(h) for h in held) == {0, 1, 2, 3, 4}
    ctx.close()


@pytest.mark.parametrize("params", [(1, 0, 0, 1), (0, 1, 0, 0), (1, 1, 1, 1), (0, 0, 1, 0)])
def test_random_pieces(R, oracle, params):
    """many pushes per stream, piece sizes from 0 to over a revolution, different for every stream; state() after
    every push"""
    n, max_nodes, max_scans = 40, 4096, 64  # a noise stretch publishes a few dozen short scans
    streams = [normal_stream(3 * NODES_PER_REV, 5000 + s, bad=s % 4 != 3) for s in range(n)]
    rng = np.random.default_rng(sum(params))
    sizes = [0, 1, 2, 3, 4, 5, 6, 7, 64, 999, 5000, 16001, 20000]
    cuts = [_random_cuts(rng, len(b), sizes) for b in streams]
    pieces, prefixes = _pieces_from_cuts(streams, cuts)
    assert any(0 < len(p) < 4 for push in pieces[:-1] for p in push)
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], max_nodes, max_scans, params)
    got, states = _run(R, ctx, pieces, max_nodes, max_scans, params, stride=20000)
    assert got == whole
    _check_oracle(oracle, got, streams, max_nodes, range(0, n, 5), params)
    which = range(0, n, 3) if params == PARAMS else range(0, n, 13)
    _check_states(oracle, states, prefixes, max_nodes, which)
    ctx.close()


def test_one_byte_per_push(R, oracle):
    """every byte boundary is a push boundary, across at least two revolution boundaries (revolutions of 40 records)"""
    n, max_nodes, max_scans, rev = 6, 4096, 2, 40
    streams = [normal_stream(130, 6000 + s, nodes_per_rev=rev, bad=s % 2 == 1, noise=9) for s in range(n)]
    m = max(len(b) for b in streams)
    pieces = [[b[t:t + 1] for b in streams] for t in range(m)]
    ctx = R.Context(0, max_nodes, n * 64)
    whole, _ = _run(R, ctx, [streams], max_nodes, 64)
    got, states = _run(R, ctx, pieces, max_nodes, max_scans, stride=1)
    assert got == whole
    assert all(len(g) >= 2 for g in got[::2])
    _check_oracle(oracle, got, streams, max_nodes, range(n))
    _check_states(oracle, states[::7], [[b[:t + 1] for b in streams] for t in range(0, m, 7)], max_nodes, range(n))
    ctx.close()


def test_short_push_after_mid_record(R, oracle):
    """a push that ends k = 0..4 bytes into a record, then a push of 0..3 bytes (the halo shifts onto itself), then
    the rest; a push of 0 bytes keeps the state"""
    b = normal_stream(2 * NODES_PER_REV + 50, 42, bad=False)
    r0 = int(np.nonzero(b[0::5] & 1)[0][0])
    cases = [(5 * r + k, m) for r in (r0 - 1, r0, r0 + 7) for k in range(0, 5) for m in range(0, 4)]
    n, max_nodes, max_scans = len(cases), 4096, 8
    streams = [b] * n
    pieces = [[b[:c] for c, _ in cases], [b[c:c + m] for c, m in cases], [b[c + m:] for c, m in cases]]
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], max_nodes, max_scans)
    got, states = _run(R, ctx, pieces, max_nodes, max_scans, stride=len(b))
    assert got == whole
    prefixes = [pieces[0], [b[:c + m] for c, m in cases], streams]
    _check_states(oracle, states, prefixes, max_nodes, range(n))
    assert (states[0][1] == np.array([c % 5 for c, _ in cases])).all()
    ctx.close()


def test_capacity_across_pushes(R, oracle):
    """max_nodes 1024 against revolutions of 3200 records, split before the cap, at it and after it"""
    n, max_nodes, max_scans = 48, 1024, 8
    streams = [normal_stream(3 * NODES_PER_REV, 7000 + s, bad=False) for s in range(n)]
    p1, p2 = [], []
    for s, b in enumerate(streams):
        r1 = int(np.nonzero(b[0::5] & 1)[0][1])  # second revolution's start record
        cut = 5 * r1 + 5 * (1 + s * 2100 // n) + s % 5  # 1 .. ~2100 records into the revolution
        p1.append(b[:cut])
        p2.append(b[cut:])
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], max_nodes, max_scans)
    got, states = _run(R, ctx, [p1, p2], max_nodes, max_scans, stride=max(len(b) for b in streams))
    assert got == whole
    _check_oracle(oracle, got, streams, max_nodes, range(0, n, 3))
    opens = states[0][0]
    assert (opens == max_nodes).any() and (opens < max_nodes).any() and (opens > 0).all()
    _check_states(oracle, states[:1], [p1], max_nodes, range(n))
    ctx.close()


def test_reset_mask(R, oracle):
    """reset while a record is half received: a reset stream continues like a fresh session fed the rest; the others
    are unaffected"""
    n, max_nodes, max_scans = 24, 4096, 64  # a noise stretch publishes a few dozen short scans
    streams = [normal_stream(2 * NODES_PER_REV, 8000 + s, bad=s % 3 == 0) for s in range(n)]
    cuts = []
    for b in streams:  # the first cut from 5/8 of the stream on where the machine holds 2 bytes
        c = len(b) * 5 // 8
        while oracle.decode_normal(b[:c])[2] != 2:
            c += 1
        cuts.append(c)
    p1, p2 = [b[:c] for b, c in zip(streams, cuts)], [b[c:] for b, c in zip(streams, cuts)]
    stride = max(len(b) for b in streams)
    ctx = R.Context(0, max_nodes, n * max_scans)
    mask = (np.arange(n) % 2 == 0)
    with R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans) as sess:
        _run(R, ctx, [p1], max_nodes, max_scans, sess=sess)
        opens0, held0 = sess.state()
        assert (held0 == 2).all() and (opens0 > 0).all()
        sess.reset(mask)
        opens, held = sess.state()
        assert (opens[mask] == 0).all() and (held[mask] == 0).all()
        assert (opens[~mask] == opens0[~mask]).all() and (held[~mask] == held0[~mask]).all()
        after, _ = _run(R, ctx, [p2], max_nodes, max_scans, sess=sess)
    fresh, _ = _run(R, ctx, [p2], max_nodes, max_scans, stride=stride)
    kept, _ = _run(R, ctx, [p1, p2], max_nodes, max_scans, stride=stride)
    kept1, _ = _run(R, ctx, [p1], max_nodes, max_scans, stride=stride)
    for s in range(n):
        if mask[s]:
            assert after[s] == fresh[s], s
        else:
            assert after[s] == kept[s][len(kept1[s]):], s
    ctx.close()


def _stateless(R, ctx, host, counts, params, max_nodes, max_scans):
    """rpl_decode_normal_batch_dev -> rpl_assemble_scan_views_dev -> rpl_scan_views_dev on the same bytes"""
    import torch

    dev = torch.device("cuda", 0)
    n, stride = host.shape
    per = stride // 5
    d_bytes = torch.from_numpy(host).to(dev)
    d_cnt = torch.from_numpy(counts.view(np.int32)).to(dev)
    nodes = torch.zeros(n * per, dtype=torch.int64, device=dev)
    node_counts = torch.zeros(n, dtype=torch.int32, device=dev)
    views = torch.zeros(n * max_scans, dtype=torch.int64, device=dev)
    scan_len = torch.zeros(n * max_scans, dtype=torch.int32, device=dev)
    sps = torch.zeros(n, dtype=torch.int32, device=dev)
    NS = n * max_scans
    r = torch.zeros((NS, max_nodes), device=dev)
    it = torch.zeros((NS, max_nodes), device=dev)
    bc = torch.zeros(NS, dtype=torch.int32, device=dev)
    inc = torch.zeros(NS, device=dev)
    torch.cuda.synchronize()
    ctx.decode_normal_batch_dev(d_bytes.data_ptr(), d_cnt.data_ptr(), n, stride, nodes.data_ptr(), node_counts.data_ptr())
    ctx.assemble_scan_views_dev(nodes.data_ptr(), node_counts.data_ptr(), n, per, max_nodes, max_scans,
                                views.data_ptr(), scan_len.data_ptr(), sps.data_ptr())
    ctx.scan_views_dev(nodes.data_ptr(), n * per, views.data_ptr(), NS, max_nodes, params, ranges=r.data_ptr(),
                       intensities=it.data_ptr(), beam_counts=bc.data_ptr(), angle_increment=inc.data_ptr())
    ctx.synchronize()
    return dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("params", [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)])
def test_first_push_equals_the_stateless_path(R, oracle, params):
    n, max_nodes, max_scans = 12, 4096, 64
    streams = [normal_stream(4 * NODES_PER_REV, 9000 + s, bad=s % 2 == 0) for s in range(n)]
    stride = max(len(b) for b in streams)
    host = np.full((n, stride), 0xEE, np.uint8)
    counts = np.zeros(n, np.uint32)
    for s, b in enumerate(streams):
        host[s, : len(b)] = b
        counts[s] = len(b)
    counts[3], counts[4], counts[5] = 0, counts[4] // 3, 4
    ctx = R.Context(0, max_nodes, n * max_scans)
    ref = _stateless(R, ctx, host, counts, R.scan_params(*params), max_nodes, max_scans)
    with R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans) as sess:
        out = sess.push(host, counts, R.scan_params(*params))
    assert _scans(out, n, max_scans) == _scans(ref, n, max_scans)
    assert (out["scans_per_stream"] == ref["scans_per_stream"]).all() and out["scans_per_stream"].sum() > n
    if params == PARAMS:
        _check_oracle(oracle, _scans(out, n, max_scans), [b[:k] for b, k in zip(streams, counts)], max_nodes,
                      range(n), params)
    ctx.close()


def test_push_dev_on_a_caller_stream_and_many_streams(R, oracle):
    """push_dev on a caller's torch stream; more streams than one chunk of the context's max_scans, so each push runs
    in several chunks; equal to the host pushes (more streams than CTAs per launch: tests/test_gpu_fleet_scale.py)"""
    import torch

    dev = torch.device("cuda", 0)
    max_nodes, max_scans = 4096, 16
    n = 8 * torch.cuda.get_device_properties(0).multi_processor_count + 37
    streams = [normal_stream(300, 10000 + s % 29, nodes_per_rev=100, bad=s % 3 == 0, noise=20) for s in range(n)]
    cut = [(7 * s) % len(b) for s, b in enumerate(streams)]
    pieces = [[b[:k] for b, k in zip(streams, cut)], [b[k:] for b, k in zip(streams, cut)]]
    stride = max(len(b) for b in streams)
    ctx = R.Context(0, max_nodes, 100 * max_scans)  # 100 streams per chunk
    ref_got, ref_states = _run(R, ctx, pieces, max_nodes, max_scans, stride=stride)
    whole, _ = _run(R, ctx, [streams], max_nodes, max_scans)
    assert ref_got == whole
    _check_oracle(oracle, ref_got, streams, max_nodes, range(0, n, 97))
    ts = torch.cuda.Stream(device=dev)
    NS = n * max_scans
    got = [[] for _ in range(n)]
    with R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans) as sess:
        for t in range(2):
            buf, cnt = _pack(pieces[t], stride)
            with torch.cuda.stream(ts):
                d_bytes = torch.from_numpy(buf).to(dev)
                d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
                r = torch.full((NS, max_nodes), -1.0, device=dev)
                it = torch.full((NS, max_nodes), -1.0, device=dev)
                bc = torch.zeros(NS, dtype=torch.int32, device=dev)
                inc = torch.zeros(NS, dtype=torch.float32, device=dev)
                sps = torch.zeros(n, dtype=torch.int32, device=dev)
            sess.push_dev(d_bytes.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=ts.cuda_stream)
            ts.synchronize()
            out = dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(),
                       beam_counts=bc.cpu().numpy().view(np.uint32), angle_increment=inc.cpu().numpy(),
                       scans_per_stream=sps.cpu().numpy().view(np.uint32))
            for s, row in enumerate(_scans(out, n, max_scans)):
                got[s] += row
            opens, held = sess.state()
            assert (opens == ref_states[t][0]).all() and (held == ref_states[t][1]).all()
    assert got == ref_got
    ctx.close()


def test_argument_checks(R):
    ctx = R.Context(0, 4096, 64)
    for max_nodes in (4095, 0, 8194):
        with pytest.raises(R.RplError) as e:
            R.NormalStreamSession(ctx, 4, 100, max_nodes, 8)
        assert e.value.code == R.RESULT_INVALID_DATA and "max_nodes" in str(e.value)
    with pytest.raises(R.RplError) as e:
        R.NormalStreamSession(ctx, 4, 100, 4096, 65)  # the context's max_scans (64) cannot cover one stream
    assert e.value.code == R.RESULT_INVALID_DATA and "max_scans" in str(e.value)
    # the 32-bit view bound: (stride_bytes + 4) / 5 rounded up to even new nodes per stream, behind max_nodes
    n_streams, max_nodes, stride = 8, 8192, 5 * (2 ** 29 - 8192) + 1
    assert n_streams * (max_nodes + (stride // 5 - 1)) < 2 ** 32 <= n_streams * (max_nodes + (((stride + 4) // 5 + 1) & ~1))
    with pytest.raises(R.RplError) as e:
        R.NormalStreamSession(ctx, n_streams, stride, max_nodes, 8)
    assert e.value.code == R.RESULT_INVALID_DATA and "2^32" in str(e.value)
    with R.NormalStreamSession(ctx, 4, 100, 4096, 8) as sess:
        counts = np.array([10, 101, 0, 5], np.uint32)
        with pytest.raises(R.RplError) as e:
            sess.push(np.zeros((4, 100), np.uint8), counts, R.scan_params(*PARAMS))
        assert e.value.code == R.RESULT_INVALID_DATA and "stride" in str(e.value)
        opens, held = sess.state()  # the refused push left the state alone
        assert (opens == 0).all() and (held == 0).all()
    ctx.close()
