"""The dense session (DenseStreamSession, rpl_capsule_stream_* on 0x85): dense capsules pushed in pieces publish exactly
the scans of the whole stream -- the SDK's unpacker -> ScanDataHolder -> ascendScanData -> publish_scan on the
concatenation (pinned on the CPU by tests/test_dense_stream_pieces.py).  Every comparison is bit for bit: against one
push of the whole stream, and against the restatement (oracle dense_decode -> assemble_scans -> ascend -> publish,
stable tie rule as in test_wire_bytes_to_laserscan_in_one_host_call) and, where oracle/_ref is built, the SDK's own
decoder and holder."""
import numpy as np
import pytest

from test_decode_oracle_vs_ref import make_stream

pytestmark = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _stream(O, n_caps, seed, sync_every=None, bad=True):
    caps = make_stream(O, n_caps, 80.0 + (seed % 7) * 0.7, seed=seed, sync_every=sync_every)
    if bad:
        rng = np.random.default_rng(seed)
        caps[rng.choice(n_caps, max(1, n_caps // 60), replace=False), 10] ^= 0x40  # checksum errors
        caps[rng.choice(n_caps, max(1, n_caps // 120), replace=False)] = 0        # bad frames (all zero)
    return caps


def _streams(O, n_streams, n_caps, seed0):
    return [_stream(O, n_caps, seed0 + s, sync_every=(150 + 7 * (s % 11)) if s % 3 else None) for s in range(n_streams)]


def _scans(out, n_streams, max_scans):
    """per stream, the published scans of one push: [(beam_count, ranges bits, intensities bits)]"""
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


def _run(R, ctx, pieces, stride, max_nodes, max_scans, params=PARAMS, sess=None):
    """pieces: list of pushes, each a list (per stream) of capsule arrays.  Returns the concatenated scans per stream
    and the state after every push."""
    n = len(pieces[0])
    own = sess is None
    sess = sess or R.DenseStreamSession(ctx, n, stride, max_nodes, max_scans)
    got, states = [[] for _ in range(n)], []
    for push in pieces:
        buf = np.zeros((n, stride, 84), np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        out = sess.push(buf, cnt, R.scan_params(*params))
        for s, row in enumerate(_scans(out, n, max_scans)):
            got[s] += row
        states.append(sess.state())
    if own:
        sess.close()
    return got, states


def _oracle_scans(O, caps, max_nodes, params=PARAMS):
    en, es, eo, _ = O.dense_decode(caps, 31, 0)
    e, el, ek = O.assemble_scans(en, O.resets_from_capsules(es, eo), max_nodes, 512)
    rows = []
    for k in range(ek):
        nodes = e[k, : el[k]].copy()
        if params[3]:
            _, nodes = O.ascend(nodes, stable=True)
        hdr, r, it = O.publish(nodes, O.scan_params(params[0], params[1], params[2], params[3], 40.0, 0.1), stable=True)
        rows.append((hdr.beam_count, r.view(np.uint32).tobytes(), it.view(np.uint32).tobytes()))
    return rows, (en, es, eo)


def _open_nodes(O, caps, max_nodes):
    """the holder's scan in progress after `caps`: nodes since the last scan start, emptied by a later reset, capped"""
    if len(caps) == 0:
        return 0
    en, es, eo, _ = O.dense_decode(caps, 31, 0)
    starts = np.nonzero(en["flag"] & 1)[0]
    if len(starts) == 0:
        return 0
    ls = int(starts[-1])
    if any(ls < int(r) <= len(en) for r in O.resets_from_capsules(es, eo)):
        return 0
    return min(len(en) - ls, max_nodes)


def _check_oracle(O, got, streams, max_nodes, which, params=PARAMS):
    for s in which:
        exp, _ = _oracle_scans(O, streams[s], max_nodes, params)
        assert len(got[s]) == len(exp), (s, len(got[s]), len(exp))
        for j, (g, e) in enumerate(zip(got[s], exp)):
            assert g[:3] == e, (s, j)


def _check_ref(O, streams, max_nodes, which):
    """where oracle/_ref is built: the SDK's own decoder and holder give the restatement's scans on these streams"""
    if not (O.have_ref() and O.have_ref_holder()):
        return
    for s in which:
        caps = streams[s]
        O.ref_dense_decode(make_stream(O, 3, 80.0, seed=1, start_deg=100.0).reshape(-1), 31, 84)  # static flag -> 0
        rn, ev = O.ref_dense_decode(caps.reshape(-1), 31, 84)
        rs, rl, rk = O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), max_nodes, 512)
        en, es, eo, _ = O.dense_decode(caps, 31, 0)
        e, el, ek = O.assemble_scans(en, O.resets_from_capsules(es, eo), max_nodes, 512)
        assert rk == ek and (rl == el).all(), s
        for k in range(min(ek, 512)):
            assert (rs[k, : rl[k]].view(np.uint64) == e[k, : el[k]].view(np.uint64)).all(), (s, k)


def test_every_split_point(R, oracle):
    """~400 streams of 400 capsules (80 per revolution, scan-reset capsules, checksum errors, all-zero capsules);
    stream s is split into two pushes at capsule s."""
    n, n_caps, max_nodes, max_scans = 400, 400, 4096, 16
    streams = _streams(oracle, n, n_caps, 7000)
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, [[c[:s] for s, c in enumerate(streams)], [c[s:] for s, c in enumerate(streams)]],
                       n_caps, max_nodes, max_scans)
    assert got == whole
    assert sum(len(g) for g in got) > 2 * n
    _check_oracle(oracle, got, streams, max_nodes, list(range(0, n, 13)) + [1, 2, 80, 81, 399])
    _check_ref(oracle, streams, max_nodes, [0, 80, 161])
    for s in range(0, n, 5):
        assert states[0][0][s] == _open_nodes(oracle, streams[s][:s], max_nodes), s
        assert states[1][0][s] == _open_nodes(oracle, streams[s], max_nodes), s
    ctx.close()


def _random_pieces(rng, n_caps):
    sizes = [0, 1, 2, 39, 40, 41, 79, 80, 81, 500]
    cuts, at = [], 0
    while at < n_caps:
        at = min(n_caps, at + int(rng.choice(sizes)))
        cuts.append(at)
    return cuts


def test_random_pieces(R, oracle):
    """many pushes per stream, piece sizes from {0, 1, 2, 39, 40, 41, 79, 80, 81, 500}, different for every stream;
    a revolution spread over three or more pushes; streams with 0 capsules in a push"""
    n, n_caps, max_nodes, max_scans = 48, 1200, 4096, 16
    streams = _streams(oracle, n, n_caps, 8000)
    rng = np.random.default_rng(5)
    cuts = [_random_pieces(rng, n_caps) for _ in range(n)]
    cuts[0] = [1, 2, 3] + list(range(40, n_caps, 20)) + [n_caps]  # one revolution over four pushes at least
    n_push = max(len(c) for c in cuts)
    pieces, bounds = [], []
    for t in range(n_push):
        push, b = [], []
        for s in range(n):
            c = [0] + cuts[s]
            lo, hi = c[min(t, len(c) - 1)], c[min(t + 1, len(c) - 1)]
            push.append(streams[s][lo:hi])
            b.append(hi)
        pieces.append(push)
        bounds.append(b)
    assert any(len(p) == 0 for push in pieces[:-1] for p in push)
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, pieces, 500, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, got, streams, max_nodes, range(n))
    for t in range(0, n_push, 3):
        for s in range(0, n, 4):
            assert states[t][0][s] == _open_nodes(oracle, streams[s][: bounds[t][s]], max_nodes), (t, s)
    ctx.close()


def test_capacity_across_pushes(R, oracle):
    """max_nodes 2048 against revolutions of 3200+ nodes, split before the cap, exactly at it and after it"""
    n, n_caps, max_nodes, max_scans = 64, 600, 2048, 8
    streams = [_stream(oracle, n_caps, 9000 + s, bad=False) for s in range(n)]
    pieces = [[], []]
    for s, c in enumerate(streams):
        en, _, eo, _ = oracle.dense_decode(c, 31, 0)
        st = int(np.nonzero(en["flag"] & 1)[0][1])  # second revolution's start node
        first_cap = int(np.searchsorted(eo, st, side="right"))  # the capsule releasing the node after it
        cut = first_cap + 40 + s  # 40..103 capsules into the revolution: 1600..4100 nodes, the cap among them
        pieces[0].append(c[:cut])
        pieces[1].append(c[cut:])
    ctx = R.Context(0, max_nodes, n * max_scans)
    whole, _ = _run(R, ctx, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, pieces, n_caps, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, got, streams, max_nodes, range(n))
    opens = states[0][0]
    assert (opens == max_nodes).any() and (opens < max_nodes).any() and (opens > 0).all()
    for s in range(n):
        assert opens[s] == _open_nodes(oracle, pieces[0][s], max_nodes), s
    ctx.close()


def test_held_capsule_and_reset_cases(R, oracle):
    """a scan-reset capsule first in a push while a revolution is open; a checksum-error or all-zero capsule last in a
    push; a push ending right after the capsule that holds a scan-start node"""
    n_caps, max_nodes, max_scans = 500, 4096, 16
    streams, cuts = [], []
    for s in range(24):
        c = _stream(oracle, n_caps, 9500 + s, bad=False)
        en, es, eo, _ = oracle.dense_decode(c, 31, 0)
        kind = s % 4
        cut = 200 + 3 * s
        if kind == 0:  # reset capsule first in the second push (a revolution is open at 200: 2.5 revolutions in)
            q6 = int(c[cut, 2]) | ((int(c[cut, 3]) & 0x7F) << 8)
            c[cut] = oracle.make_dense_capsules([q6], [True], c[cut, 4:].copy().view(np.uint16)[None, :])[0]
        elif kind == 1:  # checksum error last in the first push
            c[cut - 1, 10] ^= 0x40
        elif kind == 2:  # all-zero capsule last in the first push
            c[cut - 1] = 0
        else:  # the first push ends with the capsule holding a scan-start node (held), or with the one releasing it
            st = int(np.nonzero(en["flag"] & 1)[0][2])
            cut = int(np.searchsorted(eo, st, side="right")) - (1 if s % 8 == 3 else 0)
        streams.append(c)
        cuts.append(cut)
    pieces = [[c[:k] for c, k in zip(streams, cuts)], [c[k:] for c, k in zip(streams, cuts)]]
    ctx = R.Context(0, max_nodes, len(streams) * max_scans)
    whole, _ = _run(R, ctx, [streams], n_caps, max_nodes, max_scans)
    got, states = _run(R, ctx, pieces, n_caps, max_nodes, max_scans)
    assert got == whole
    _check_oracle(oracle, got, streams, max_nodes, range(len(streams)))
    opens, held = states[0]
    for s in range(len(streams)):
        assert opens[s] == _open_nodes(oracle, pieces[0][s], max_nodes), s
        assert held[s] == (0 if s % 4 in (1, 2) else 1), s
    assert (states[1][0][0::4] == [_open_nodes(oracle, c, max_nodes) for c in streams[0::4]]).all()
    ctx.close()


@pytest.mark.parametrize("params", [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)])
def test_first_push_equals_the_chain(R, oracle, params):
    n, n_caps, max_nodes, max_scans = 24, 700, 4096, 12
    streams = _streams(oracle, n, n_caps, 10000)
    ctx = R.Context(0, max_nodes, n * max_scans)
    host = np.stack(streams)
    counts = np.full(n, n_caps, np.uint32)
    counts[3], counts[4] = 0, 77
    chain = ctx.chain_dense_laserscan(host, counts, R.scan_params(*params), max_nodes, max_scans)
    with R.DenseStreamSession(ctx, n, n_caps, max_nodes, max_scans) as sess:
        out = sess.push(host, counts, R.scan_params(*params))
    for k in ("ranges", "intensities", "beam_counts", "angle_increment", "scans_per_stream"):
        assert (out[k].view(np.uint32) == chain[k].view(np.uint32)).all(), k
    ctx.close()


def test_reset_mask(R, oracle):
    """a reset stream continues like a fresh session fed the rest; the others are unaffected"""
    n, n_caps, max_nodes, max_scans = 32, 600, 4096, 16
    streams = _streams(oracle, n, n_caps, 11000)
    p1, p2 = [c[:250] for c in streams], [c[250:] for c in streams]
    ctx = R.Context(0, max_nodes, n * max_scans)
    mask = (np.arange(n) % 2 == 0)
    with R.DenseStreamSession(ctx, n, n_caps, max_nodes, max_scans) as sess:
        _run(R, ctx, [p1], n_caps, max_nodes, max_scans, sess=sess)
        sess.reset(mask)
        opens, held = sess.state()
        assert (opens[mask] == 0).all() and (held[mask] == 0).all() and (held[~mask] == 1).any()
        after, _ = _run(R, ctx, [p2], n_caps, max_nodes, max_scans, sess=sess)
    fresh, _ = _run(R, ctx, [p2], n_caps, max_nodes, max_scans)
    kept, _ = _run(R, ctx, [p1, p2], n_caps, max_nodes, max_scans)
    kept2, _ = _run(R, ctx, [p1], n_caps, max_nodes, max_scans)
    for s in range(n):
        if mask[s]:
            assert after[s] == fresh[s], s
        else:
            assert after[s] == kept[s][len(kept2[s]):], s
    ctx.close()


def test_two_sessions_push_dev_and_many_streams(R, oracle):
    """two sessions pushed alternately on one context; push_dev on a caller's non-default torch stream equals push;
    more streams than one chunk, so each push runs in several chunks (more streams than CTAs per launch:
    tests/test_gpu_fleet_scale.py)"""
    import torch

    n_caps, max_nodes, max_scans = 240, 4096, 8
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 37
    streams = _streams(oracle, n, n_caps, 12000)
    cut = [60 + s % 97 for s in range(n)]
    pieces = [[c[:k] for c, k in zip(streams, cut)], [c[k:] for c, k in zip(streams, cut)]]
    ctx = R.Context(0, max_nodes, 100 * max_scans)  # 100 streams per chunk
    ref_got, ref_states = _run(R, ctx, pieces, n_caps, max_nodes, max_scans)
    whole, _ = _run(R, ctx, [streams], n_caps, max_nodes, max_scans)
    assert ref_got == whole
    _check_oracle(oracle, ref_got, streams, max_nodes, range(0, n, 41))
    # two sessions, alternating pushes (the second one fed the pieces in reverse stream order)
    a = R.DenseStreamSession(ctx, n, n_caps, max_nodes, max_scans)
    b = R.DenseStreamSession(ctx, n, n_caps, max_nodes, max_scans)
    ga, gb = [[] for _ in range(n)], [[] for _ in range(n)]
    for push in pieces:
        for sess, g, order in ((a, ga, 1), (b, gb, -1)):
            ps = push[::order]
            buf = np.zeros((n, n_caps, 84), np.uint8)
            cnt = np.array([len(p) for p in ps], np.uint32)
            for s, p in enumerate(ps):
                buf[s, : len(p)] = p
            for s, row in enumerate(_scans(sess.push(buf, cnt, R.scan_params(*PARAMS)), n, max_scans)):
                g[s] += row
    assert ga == ref_got and gb == ref_got[::-1]
    a.close()
    b.close()
    # push_dev on a torch stream
    dev = torch.device("cuda", 0)
    sess = R.DenseStreamSession(ctx, n, n_caps, max_nodes, max_scans)
    ts = torch.cuda.Stream(device=dev)
    got = [[] for _ in range(n)]
    for t, push in enumerate(pieces):
        buf = np.zeros((n, n_caps, 84), np.uint8)
        cnt = np.array([len(p) for p in push], np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
        NS = n * max_scans
        with torch.cuda.stream(ts):
            d_caps = torch.from_numpy(buf).to(dev, non_blocking=False)
            d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
            r = torch.full((NS, max_nodes), -1.0, device=dev)
            it = torch.full((NS, max_nodes), -1.0, device=dev)
            bc = torch.zeros(NS, dtype=torch.int32, device=dev)
            inc = torch.zeros(NS, dtype=torch.float32, device=dev)
            sps = torch.zeros(n, dtype=torch.int32, device=dev)
        sess.push_dev(d_caps.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS), r.data_ptr(), it.data_ptr(),
                      bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=ts.cuda_stream)
        ts.synchronize()
        out = dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                   angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32))
        for s, row in enumerate(_scans(out, n, max_scans)):
            got[s] += row
        opens, held = sess.state()
        assert (opens == ref_states[t][0]).all() and (held == ref_states[t][1]).all()
    assert got == ref_got
    sess.close()
    ctx.close()


def test_argument_checks(R):
    ctx = R.Context(0, 4096, 64)
    for max_nodes in (4095, 0, 8194):
        with pytest.raises(R.RplError) as e:
            R.DenseStreamSession(ctx, 4, 100, max_nodes, 8)
        assert e.value.code == R.RESULT_INVALID_DATA and "max_nodes" in str(e.value)
    with pytest.raises(R.RplError) as e:
        R.DenseStreamSession(ctx, 4, 100, 4096, 65)  # the context's max_scans (64) cannot cover one stream
    assert e.value.code == R.RESULT_INVALID_DATA and "max_scans" in str(e.value)
    with R.DenseStreamSession(ctx, 4, 100, 4096, 8) as sess:
        counts = np.array([10, 101, 0, 5], np.uint32)
        with pytest.raises(R.RplError) as e:
            sess.push(np.zeros((4, 100, 84), np.uint8), counts, R.scan_params(*PARAMS))
        assert e.value.code == R.RESULT_INVALID_DATA and "stride" in str(e.value)
        opens, held = sess.state()  # the refused push left the state alone
        assert (opens == 0).all() and (held == 0).all()
    ctx.close()
