"""rpl_capsule_stream_* (CapsuleStreamSession) for express (0x82), HQ (0x83), ultra (0x84) and ultra-dense (0x86)
capsules: a stream pushed in pieces publishes exactly the scans of the whole stream -- the SDK's unpacker ->
ScanDataHolder -> ascendScanData -> publish_scan on the concatenation (pinned on the CPU by
tests/test_capsule_stream_pieces.py).  Every comparison is bit for bit on ranges, intensities, beam counts and angle
increment: against one push of the whole stream, against the restatement (oracle decode_capsules -> assemble_scans ->
ascend -> publish, stable tie rule) and, where oracle/_ref is built, the SDK's own decoder and holder.  The dense
format's session is tests/test_gpu_dense_stream.py; here it is only checked to be the same session."""
import numpy as np
import pytest

from test_capsule_stream_pieces import STREAM_FORMATS, format_stream, hq_capsules, restated_scans
from test_decode_oracle_vs_ref import make_stream

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
# capsules per stream for about 12800 nodes (4.5 revolutions) in every format
N_CAPS = {0x82: 400, 0x83: 134, 0x84: 134, 0x86: 200}
CAPS_PER_REV = {0x82: 80, 0x83: 30, 0x84: 30, 0x86: 45}


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _streams(O, ans, n, n_caps, seed0, bad=True):
    """streams of one format; every third without scan-start capsules, every other ultra-dense one with the smoothing
    chain's short-range samples"""
    return [format_stream(O, ans, n_caps, seed0 + s, sync_every=(250 + 7 * (s % 11)) if s % 3 else None, bad=bad,
                          near=(ans == 0x86 and s % 2 == 0)) for s in range(n)]


def _scans(out, n_streams, max_scans):
    """per stream, the published scans of one push: [(beam_count, ranges bits, intensities bits, increment bits)]"""
    res = []
    for s in range(n_streams):
        k = int(out["scans_per_stream"][s])
        assert k <= max_scans, (s, k)
        row = []
        for j in range(k):
            slot = s * max_scans + j
            m = int(out["beam_counts"][slot])
            row.append((m, out["ranges"][slot, :m].view(np.uint32).tobytes(),
                        out["intensities"][slot, :m].view(np.uint32).tobytes(),
                        out["angle_increment"][slot:slot + 1].view(np.uint32).tobytes()))
        res.append(row)
    return res


def _pack(push, stride, cb):
    n = len(push)
    buf = np.zeros((n, stride, cb), np.uint8)
    cnt = np.zeros(n, np.uint32)
    for s, p in enumerate(push):
        buf[s, : len(p)] = p
        cnt[s] = len(p)
    return buf, cnt


def _run(R, ctx, ans, pieces, stride, max_nodes, max_scans, params=PARAMS, sess=None):
    """pieces: list of pushes, each a list (per stream) of capsule arrays.  Returns the concatenated scans per stream
    and the state after every push."""
    n = len(pieces[0])
    own = sess is None
    sess = sess or R.CapsuleStreamSession(ctx, ans, n, stride, max_nodes, max_scans)
    got, states = [[] for _ in range(n)], []
    for push in pieces:
        buf, cnt = _pack(push, stride, sess.capsule_bytes)
        out = sess.push(buf, cnt, R.scan_params(*params))
        for s, row in enumerate(_scans(out, n, max_scans)):
            got[s] += row
        states.append(sess.state())
    if own:
        sess.close()
    return got, states


def _oracle_rows(O, ans, caps, max_nodes, params=PARAMS):
    e, el, ek, _, _, _ = restated_scans(O, ans, caps, max_nodes)
    rows = []
    for k in range(ek):
        nodes = e[k, : el[k]].copy()
        if params[3]:
            _, nodes = O.ascend(nodes, stable=True)
        hdr, r, it = O.publish(nodes, O.scan_params(params[0], params[1], params[2], params[3], 40.0, 0.1), stable=True)
        rows.append((hdr.beam_count, r.view(np.uint32).tobytes(), it.view(np.uint32).tobytes()))
    return rows


def _expected_state(O, ans, caps, max_nodes):
    """(open nodes, held capsule) after `caps`: the holder's scan in progress (nodes since the last scan start, emptied
    by a later reset, capped), and whether the last capsule is a valid one held back (never for HQ)"""
    if len(caps) == 0:
        return 0, 0
    nodes, status, offs, _ = O.decode_capsules(ans, caps, 31)
    held = 0 if ans == 0x83 else int((status[-1] & O.CAPSULE_OK) != 0)
    starts = np.nonzero(nodes["flag"] & 1)[0]
    if len(starts) == 0:
        return 0, held
    ls = int(starts[-1])
    if any(ls < int(r) <= len(nodes) for r in O.resets_from_capsules(status, offs)):
        return 0, held
    return min(len(nodes) - ls, max_nodes), held


def _check_states(O, ans, states, prefixes, max_nodes, which):
    """states[t] after push t against the restatement on prefixes[t][s] (the capsules pushed so far)"""
    for t, st in enumerate(states):
        for s in which:
            exp = _expected_state(O, ans, prefixes[t][s], max_nodes)
            assert (int(st[0][s]), int(st[1][s])) == exp, (t, s)


def _check_oracle(O, ans, got, streams, max_nodes, which, params=PARAMS):
    for s in which:
        exp = _oracle_rows(O, ans, streams[s], max_nodes, params)
        assert len(got[s]) == len(exp), (s, len(got[s]), len(exp))
        for j, (g, e) in enumerate(zip(got[s], exp)):
            assert g[:3] == e, (s, j)


def _check_ref(O, ans, streams, max_nodes, which):
    """where oracle/_ref is built: the SDK's own decoder and holder give the restatement's scans on these streams"""
    if not (O.have_ref() and O.have_ref_holder()):
        return
    for s in which:
        rn, ev = O.ref_unpack(ans, streams[s].reshape(-1), 31, 0)
        rs, rl, rk = O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), max_nodes, 512)
        e, el, ek, _, _, _ = restated_scans(O, ans, streams[s], max_nodes)
        assert rk == ek and (rl == el).all(), s
        for k in range(min(ek, 512)):
            assert (rs[k, : rl[k]].view(np.uint64) == e[k, : el[k]].view(np.uint64)).all(), (s, k)


@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_every_split_point(R, oracle, ans):
    """stream s is split into two pushes at capsule s: every split point of the stream, each in its own stream"""
    n_caps, max_nodes, max_scans = N_CAPS[ans], 4096, 16
    n = n_caps + 1
    streams = _streams(oracle, ans, n, n_caps, 7000)
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, max_scans)
    p1, p2 = [c[:s] for s, c in enumerate(streams)], [c[s:] for s, c in enumerate(streams)]
    got, states = _run(R, ctx, ans, [p1, p2], n_caps, max_nodes, max_scans)
    assert got == whole
    assert sum(len(g) for g in got) > 2 * n
    _check_oracle(oracle, ans, got, streams, max_nodes, list(range(0, n, 11)) + [1, 2, n - 2, n - 1])
    _check_ref(oracle, ans, streams, max_nodes, [0, 1, 5])
    _check_states(oracle, ans, states, [p1, streams], max_nodes, range(0, n, 5))
    ctx.close()


def _random_cuts(rng, n_caps, sizes):
    cuts, at = [], 0
    while at < n_caps:
        at = min(n_caps, at + int(rng.choice(sizes)))
        cuts.append(at)
    return cuts


def _pieces_from_cuts(streams, cuts):
    n_push = max(len(c) for c in cuts)
    pieces, prefixes = [], []
    for t in range(n_push):
        push, pre = [], []
        for s, cs in enumerate(cuts):
            c = [0] + cs
            lo, hi = c[min(t, len(c) - 1)], c[min(t + 1, len(c) - 1)]
            push.append(streams[s][lo:hi])
            pre.append(streams[s][:hi])
        pieces.append(push)
        prefixes.append(pre)
    return pieces, prefixes


@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_random_pieces(R, oracle, ans):
    """many pushes per stream, piece sizes around a revolution and down to 0 and 1 capsules, different for every stream;
    a revolution spread over three or more pushes"""
    n, max_nodes, max_scans = 40, 4096, 16
    n_caps, rev = 3 * N_CAPS[ans], CAPS_PER_REV[ans]
    streams = _streams(oracle, ans, n, n_caps, 8000)
    rng = np.random.default_rng(ans)
    stride = 2 * rev + 2
    sizes = [0, 1, 2, rev // 3, rev - 1, rev, rev + 1, 2 * rev + 2]
    cuts = [_random_cuts(rng, n_caps, sizes) for _ in range(n)]
    cuts[0] = [1, 2, 3] + list(range(rev // 4 + 3, n_caps, max(1, rev // 4))) + [n_caps]
    pieces, prefixes = _pieces_from_cuts(streams, cuts)
    assert any(len(p) == 0 for push in pieces[:-1] for p in push)
    assert any(len(p) == 1 for push in pieces[:-1] for p in push)
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, ans, pieces, stride, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, ans, got, streams, max_nodes, range(0, n, 3))
    _check_states(oracle, ans, states[::4], prefixes[::4], max_nodes, range(0, n, 4))
    ctx.close()


def _hq_start_capsules(caps):
    flags = caps[:, 9:9 + 768].reshape(len(caps), 96, 8)[:, :, 7]
    return np.nonzero((flags & 1).any(axis=1))[0]


@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_push_ends_on_error_zero_frame_or_scan_start(R, oracle, ans):
    """the first push ends on a checksum / CRC error, on an all-zero frame, on a scan-start capsule (HQ: the capsule
    holding a revolution's first node), or just before one -- so that the second push begins with it"""
    n_caps, max_nodes, max_scans = N_CAPS[ans], 4096, 16
    streams, cuts = [], []
    for s in range(32):
        k0 = 30 + 3 * s  # a scan-start capsule every k0, the first push ends at (or just before) the second
        c = format_stream(oracle, ans, n_caps, 9500 + s, sync_every=k0, bad=False)
        kind = s % 4
        if ans == 0x83:
            k0 = int(_hq_start_capsules(c)[1])
        cut = k0 + 1
        if kind == 0:
            c[cut - 1, 20] ^= 0x08  # checksum / CRC error last in the first push
        elif kind == 1:
            c[cut - 1] = 0  # all-zero frame last in the first push
        elif kind == 3:
            cut = k0  # the scan-start capsule opens the second push
        streams.append(c)
        cuts.append(cut)
    p1, p2 = [c[:k] for c, k in zip(streams, cuts)], [c[k:] for c, k in zip(streams, cuts)]
    ctx = R.Context(0, max_nodes, len(streams) * max_scans)
    whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, ans, [p1, p2], n_caps, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, ans, got, streams, max_nodes, range(len(streams)))
    _check_states(oracle, ans, states, [p1, streams], max_nodes, range(len(streams)))
    held = states[0][1]
    assert (held == 0).all() if ans == 0x83 else ((held[0::4] == 0).all() and (held[1::4] == 0).all()
                                                  and (held[2::4] == 1).all() and (held[3::4] == 1).all())
    ctx.close()


@pytest.mark.parametrize("ans", [0x84, 0x86])
def test_one_capsule_per_push(R, oracle, ans):
    """every capsule boundary is a push boundary.  Ultra: the held capsule's last cabin reads cabin 0 of the next
    push's first capsule.  Ultra-dense: the smoothing chain crosses every boundary, and so does the "not twice in a
    row" scan-start rule (scan starts on a capsule's last node are counted, so the case is known to occur)."""
    n, n_caps, max_nodes, max_scans = 48, 2 * N_CAPS[ans], 4096, 4
    streams = _streams(oracle, ans, n, n_caps, 9700, bad=True)
    per = oracle.capsule_nodes(ans)
    if ans == 0x86:
        last_node_starts = 0
        for c in streams:
            nodes, _, offs, _ = oracle.decode_capsules(ans, c, 31)
            idx = np.nonzero(nodes["flag"] & 1)[0]
            last_node_starts += int(((idx % per) == per - 1).sum())
        assert last_node_starts > 0
    pieces = [[c[t:t + 1] for c in streams] for t in range(n_caps)]
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, 64)
    got, states = _run(R, ctx, ans, pieces, 1, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, ans, got, streams, max_nodes, range(0, n, 5))
    _check_states(oracle, ans, states[::37], [[c[:t + 1] for c in streams] for t in range(0, n_caps, 37)], max_nodes,
                  range(0, n, 7))
    ctx.close()


@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_capacity_across_pushes(R, oracle, ans):
    """max_nodes 1024 against revolutions of about 2600-2900 nodes, split before the cap, at it and after it"""
    n, max_nodes, max_scans = 48, 1024, 8
    n_caps, per = N_CAPS[ans], oracle.capsule_nodes(ans)
    streams = _streams(oracle, ans, n, n_caps, 9000, bad=False)
    pieces = [[], []]
    for s, c in enumerate(streams):
        nodes, _, offs, _ = oracle.decode_capsules(ans, c, 31)
        st = int(np.nonzero(nodes["flag"] & 1)[0][1])  # second revolution's start node
        first_cap = int(np.searchsorted(offs, st, side="right"))  # the capsule releasing the node after it
        cut = first_cap + (1 + s * 2048 // (n * per))  # 0 .. ~2100 nodes into the revolution
        pieces[0].append(c[:cut])
        pieces[1].append(c[cut:])
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, ans, pieces, n_caps, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, ans, got, streams, max_nodes, range(n))
    opens = states[0][0]
    assert (opens == max_nodes).any() and (opens < max_nodes).any() and (opens > 0).all()
    _check_states(oracle, ans, states[:1], [pieces[0]], max_nodes, range(n))
    ctx.close()


@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_reset_mask(R, oracle, ans):
    """a reset stream continues like a fresh session fed the rest; the others are unaffected"""
    n, max_nodes, max_scans = 24, 4096, 16
    n_caps = N_CAPS[ans]
    streams = _streams(oracle, ans, n, n_caps, 11000)
    k = n_caps * 5 // 8
    p1, p2 = [c[:k] for c in streams], [c[k:] for c in streams]
    ctx = R.Context(0, max_nodes, n * max_scans)
    mask = (np.arange(n) % 2 == 0)
    with R.CapsuleStreamSession(ctx, ans, n, n_caps, max_nodes, max_scans) as sess:
        _run(R, ctx, ans, [p1], n_caps, max_nodes, max_scans, sess=sess)
        opens0, held0 = sess.state()
        sess.reset(mask)
        opens, held = sess.state()
        assert (opens[mask] == 0).all() and (held[mask] == 0).all()
        assert (opens[~mask] == opens0[~mask]).all() and (held[~mask] == held0[~mask]).all() and (opens0 > 0).any()
        assert ans == 0x83 or (held0[~mask] == 1).any()
        after, _ = _run(R, ctx, ans, [p2], n_caps, max_nodes, max_scans, sess=sess)
    fresh, _ = _run(R, ctx, ans, [p2], n_caps, max_nodes, max_scans)
    kept, _ = _run(R, ctx, ans, [p1, p2], n_caps, max_nodes, max_scans)
    kept1, _ = _run(R, ctx, ans, [p1], n_caps, max_nodes, max_scans)
    for s in range(n):
        if mask[s]:
            assert after[s] == fresh[s], s
        else:
            assert after[s] == kept[s][len(kept1[s]):], s
    ctx.close()


def _stateless(R, ctx, ans, host, counts, params, max_nodes, max_scans):
    """rpl_decode_capsules_batch_dev -> rpl_assemble_scan_views_dev -> rpl_scan_views_dev on the same capsules"""
    import torch

    dev = torch.device("cuda", 0)
    n, stride, _ = host.shape
    per = int(R.lib().rpl_capsule_nodes(ans))
    d_caps = torch.from_numpy(host).to(dev)
    d_cnt = torch.from_numpy(counts.view(np.int32)).to(dev)
    nodes = torch.zeros(n * stride * per, dtype=torch.int64, device=dev)
    node_counts = torch.zeros(n, dtype=torch.int32, device=dev)
    status = torch.zeros(n * stride, dtype=torch.int32, device=dev)
    offs = torch.zeros(n * stride, dtype=torch.int32, device=dev)
    views = torch.zeros(n * max_scans, dtype=torch.int64, device=dev)
    scan_len = torch.zeros(n * max_scans, dtype=torch.int32, device=dev)
    sps = torch.zeros(n, dtype=torch.int32, device=dev)
    NS = n * max_scans
    r = torch.zeros((NS, max_nodes), device=dev)
    it = torch.zeros((NS, max_nodes), device=dev)
    bc = torch.zeros(NS, dtype=torch.int32, device=dev)
    inc = torch.zeros(NS, device=dev)
    ctx.decode_capsules_batch_dev(ans, d_caps.data_ptr(), d_cnt.data_ptr(), n, stride, 31, nodes.data_ptr(),
                                  node_counts.data_ptr(), capsule_status=status.data_ptr(),
                                  capsule_node_offset=offs.data_ptr())
    ctx.assemble_scan_views_dev(nodes.data_ptr(), node_counts.data_ptr(), n, stride * per, max_nodes, max_scans,
                                views.data_ptr(), scan_len.data_ptr(), sps.data_ptr(), capsule_status=status.data_ptr(),
                                capsule_node_offset=offs.data_ptr(), capsule_counts=d_cnt.data_ptr(),
                                stride_capsules=stride)
    ctx.scan_views_dev(nodes.data_ptr(), n * stride * per, views.data_ptr(), NS, max_nodes, params,
                       ranges=r.data_ptr(), intensities=it.data_ptr(), beam_counts=bc.data_ptr(),
                       angle_increment=inc.data_ptr())
    torch.cuda.synchronize()
    return dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("params", [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)])
@pytest.mark.parametrize("ans", STREAM_FORMATS)
def test_first_push_equals_the_stateless_path(R, oracle, ans, params):
    n, max_nodes, max_scans = 12, 4096, 12
    n_caps = N_CAPS[ans]
    streams = _streams(oracle, ans, n, n_caps, 10000)
    ctx = R.Context(0, max_nodes, n * max_scans)
    host = np.ascontiguousarray(np.stack(streams))
    counts = np.full(n, n_caps, np.uint32)
    counts[3], counts[4] = 0, n_caps // 3
    ref = _stateless(R, ctx, ans, host, counts, R.scan_params(*params), max_nodes, max_scans)
    with R.CapsuleStreamSession(ctx, ans, n, n_caps, max_nodes, max_scans) as sess:
        out = sess.push(host, counts, R.scan_params(*params))
    assert _scans(out, n, max_scans) == _scans(ref, n, max_scans)
    assert (out["scans_per_stream"] == ref["scans_per_stream"]).all() and out["scans_per_stream"].sum() > n
    if params == (1, 0, 0, 1):
        _check_oracle(oracle, ans, _scans(out, n, max_scans), [c[:k] for c, k in zip(streams, counts)], max_nodes,
                      range(n), params)
    ctx.close()


def test_two_formats_push_dev_and_many_streams(R, oracle):
    """an ultra and an ultra-dense session pushed alternately with push_dev on a caller's torch stream, on one context;
    more streams than one chunk of the context's max_scans, so each push runs in several chunks; both equal their host
    pushes (more streams than CTAs per launch: tests/test_gpu_fleet_scale.py)"""
    import torch

    dev = torch.device("cuda", 0)
    max_nodes, max_scans = 4096, 8
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 37
    ctx = R.Context(0, max_nodes, 100 * max_scans)  # 100 streams per chunk
    fmt = {}
    for ans in (0x84, 0x86):
        n_caps = N_CAPS[ans] // 2
        streams = [format_stream(oracle, ans, n_caps, 12000 + s % 23, sync_every=None if s % 3 else 40)
                   for s in range(n)]
        cut = [(7 + s) % n_caps for s in range(n)]
        pieces = [[c[:k] for c, k in zip(streams, cut)], [c[k:] for c, k in zip(streams, cut)]]
        ref_got, ref_states = _run(R, ctx, ans, pieces, n_caps, max_nodes, max_scans)
        whole, _ = _run(R, ctx, ans, [streams], n_caps, max_nodes, max_scans)
        assert ref_got == whole
        _check_oracle(oracle, ans, ref_got, streams, max_nodes, range(0, n, 41))
        fmt[ans] = (n_caps, pieces, ref_got, ref_states, R.CapsuleStreamSession(ctx, ans, n, n_caps, max_nodes, max_scans),
                    [[] for _ in range(n)])
    ts = torch.cuda.Stream(device=dev)
    NS = n * max_scans
    for t in range(2):
        for ans, (n_caps, pieces, ref_got, ref_states, sess, got) in fmt.items():
            buf, cnt = _pack(pieces[t], n_caps, sess.capsule_bytes)
            with torch.cuda.stream(ts):
                d_caps = torch.from_numpy(buf).to(dev)
                d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
                r = torch.full((NS, max_nodes), -1.0, device=dev)
                it = torch.full((NS, max_nodes), -1.0, device=dev)
                bc = torch.zeros(NS, dtype=torch.int32, device=dev)
                inc = torch.zeros(NS, dtype=torch.float32, device=dev)
                sps = torch.zeros(n, dtype=torch.int32, device=dev)
            sess.push_dev(d_caps.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=ts.cuda_stream)
            ts.synchronize()
            out = dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(),
                       beam_counts=bc.cpu().numpy().view(np.uint32), angle_increment=inc.cpu().numpy(),
                       scans_per_stream=sps.cpu().numpy().view(np.uint32))
            for s, row in enumerate(_scans(out, n, max_scans)):
                got[s] += row
            opens, held = sess.state()
            assert (opens == ref_states[t][0]).all() and (held == ref_states[t][1]).all()
    for ans, (_, _, ref_got, _, sess, got) in fmt.items():
        assert got == ref_got, ans
        sess.close()
    ctx.close()


def test_dense_capsule_session_is_the_dense_session(R, oracle):
    """rpl_capsule_stream_create(..., 0x85, ...) publishes what DenseStreamSession publishes, push for push"""
    n, n_caps, max_nodes, max_scans = 40, 500, 4096, 16
    streams = [make_stream(oracle, n_caps, 80.0 + s % 5, seed=13000 + s, sync_every=(190 + s) if s % 2 else None)
               for s in range(n)]
    for c in streams[::3]:
        c[n_caps // 3, 10] ^= 0x40
    rng = np.random.default_rng(3)
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, n_caps, [0, 1, 39, 40, 41, 120]) for _ in range(n)])
    ctx = R.Context(0, max_nodes, n * max_scans)
    with R.CapsuleStreamSession(ctx, 0x85, n, 120, max_nodes, max_scans) as a, \
            R.DenseStreamSession(ctx, n, 120, max_nodes, max_scans) as b:
        for push in pieces:
            buf, cnt = _pack(push, 120, 84)
            oa, ob = a.push(buf, cnt, R.scan_params(*PARAMS)), b.push(buf, cnt, R.scan_params(*PARAMS))
            assert _scans(oa, n, max_scans) == _scans(ob, n, max_scans)
            assert (oa["scans_per_stream"] == ob["scans_per_stream"]).all()
            sa, sb = a.state(), b.state()
            assert (sa[0] == sb[0]).all() and (sa[1] == sb[1]).all()
    ctx.close()


def test_argument_checks(R):
    ctx = R.Context(0, 4096, 64)
    for ans in (0x81, 0x00, 0x87):
        with pytest.raises(R.RplError) as e:
            R.CapsuleStreamSession(ctx, ans, 4, 100, 4096, 8)
        assert e.value.code == R.RESULT_INVALID_DATA and "0x82..0x86" in str(e.value)
    for max_nodes in (4095, 0, 8194):
        with pytest.raises(R.RplError) as e:
            R.CapsuleStreamSession(ctx, 0x84, 4, 100, max_nodes, 8)
        assert e.value.code == R.RESULT_INVALID_DATA and "max_nodes" in str(e.value)
    with pytest.raises(R.RplError) as e:
        R.CapsuleStreamSession(ctx, 0x86, 4, 100, 4096, 65)  # the context's max_scans (64) cannot cover one stream
    assert e.value.code == R.RESULT_INVALID_DATA and "max_scans" in str(e.value)
    # the 32-bit view bound counts the format's nodes per capsule: 96 for ultra and HQ, where dense has 40
    n_streams, stride, max_nodes = 8, 5600000, 8192
    assert n_streams * (max_nodes + 40 * stride) < 2 ** 32 <= n_streams * (max_nodes + 96 * stride)
    for ans in (0x83, 0x84):
        with pytest.raises(R.RplError) as e:
            R.CapsuleStreamSession(ctx, ans, n_streams, stride, max_nodes, 8)
        assert e.value.code == R.RESULT_INVALID_DATA and "2^32" in str(e.value)
    for ans in STREAM_FORMATS:
        cb = int(R.lib().rpl_capsule_bytes(ans))
        with R.CapsuleStreamSession(ctx, ans, 4, 100, 4096, 8) as sess:
            counts = np.array([10, 101, 0, 5], np.uint32)
            with pytest.raises(R.RplError) as e:
                sess.push(np.zeros((4, 100, cb), np.uint8), counts, R.scan_params(*PARAMS))
            assert e.value.code == R.RESULT_INVALID_DATA and "stride" in str(e.value)
            opens, held = sess.state()  # the refused push left the state alone
            assert (opens == 0).all() and (held == 0).all()
    ctx.close()
