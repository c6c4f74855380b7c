"""GPU tests of scan assembly (SURVEY.md 8(f) rank 2) against the restatement orc_assemble_scans,
which tests/test_decode_oracle_vs_ref.py pins against the reference's own ScanDataHolder.
Index/byte work: bit-exact."""
import numpy as np
import pytest

from test_decode_oracle_vs_ref import make_stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 40000, 64)
    yield c
    c.close()


def random_stream(oracle, rng, n, p_sync, n_resets):
    nodes = np.zeros(n, oracle.NODE_DTYPE)
    nodes["angle_z_q14"] = rng.integers(0, 65536, n)
    nodes["dist_mm_q2"] = rng.integers(0, 1 << 20, n)
    nodes["quality"] = rng.integers(0, 256, n)
    sync = rng.random(n) < p_sync
    nodes["flag"] = np.where(sync, 1, 2)
    resets = np.sort(rng.integers(0, n + 1, n_resets)).astype(np.uint32) if n else np.zeros(0, np.uint32)
    return nodes, resets


def run_gpu(ctx, oracle, streams, max_nodes, max_scans, with_resets=True):
    """streams: list of (nodes, resets).  The resets travel as a fake decoder report: one SYNC
    capsule per reset at that node offset, interleaved with plain capsules."""
    import torch

    dev = torch.device("cuda")
    S = len(streams)
    stride = max(max(len(n) for n, _ in streams), 1)
    cstride = max(max(2 * len(r) for _, r in streams), 1)
    hn = np.zeros((S, stride), oracle.NODE_DTYPE)
    hc = np.zeros(S, np.uint32)
    hst = np.zeros((S, cstride), np.uint32)
    hof = np.zeros((S, cstride), np.uint32)
    hcc = np.zeros(S, np.uint32)
    for s, (n, r) in enumerate(streams):
        hn[s, : len(n)] = n
        hc[s] = len(n)
        # every reset capsule is followed by a plain capsule at the same offset (must not count)
        hst[s, 0: 2 * len(r): 2] = 2 | 1
        hst[s, 1: 2 * len(r): 2] = 1
        hof[s, 0: 2 * len(r): 2] = r
        hof[s, 1: 2 * len(r): 2] = r
        hcc[s] = 2 * len(r)
    t = lambda a: torch.from_numpy(a.view(np.uint8) if a.dtype == oracle.NODE_DTYPE else a.view(np.int32)).to(dev)
    nodes, counts, st, of, cc = t(hn), t(hc), t(hst), t(hof), t(hcc)
    scans = torch.zeros((S, max_scans, max_nodes, 8), dtype=torch.uint8, device=dev)
    slen = torch.zeros((S, max_scans), dtype=torch.int32, device=dev)
    sps = torch.zeros(S, dtype=torch.int32, device=dev)
    kw = dict(capsule_status=st.data_ptr(), capsule_node_offset=of.data_ptr(), capsule_counts=cc.data_ptr(),
              stride_capsules=cstride) if with_resets else {}
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.assemble_scans_dev(nodes.data_ptr(), counts.data_ptr(), S, stride, max_nodes, max_scans, max_nodes,
                           scans.data_ptr(), slen.data_ptr(), sps.data_ptr(), **kw)
    ctx.synchronize()
    torch.cuda.synchronize()
    g = scans.cpu().numpy().view(oracle.NODE_DTYPE).reshape(S, max_scans, max_nodes)
    return g, slen.cpu().numpy().astype(np.uint32), sps.cpu().numpy().astype(np.uint32)


def compare(oracle, streams, got, max_nodes, max_scans, with_resets=True):
    g, glen, gk = got
    for s, (n, r) in enumerate(streams):
        e, elen, ek = oracle.assemble_scans(n, r if with_resets else None, max_nodes, max_scans)
        assert gk[s] == ek, (s, gk[s], ek)
        for k in range(min(ek, max_scans)):
            assert glen[s, k] == elen[k], (s, k)
            assert (g[s, k, : elen[k]].view(np.uint64) == e[k, : elen[k]].view(np.uint64)).all(), (s, k)


@pytest.mark.parametrize("with_resets", [True, False])
def test_random_streams(R, oracle, ctx, with_resets):
    rng = np.random.default_rng(17)
    streams = [random_stream(oracle, rng, int(rng.integers(0, 3000)), float(rng.choice([0.002, 0.01, 0.05, 0.5])),
                             int(rng.integers(0, 12))) for _ in range(96)]
    streams += [random_stream(oracle, rng, n, 0.3, 3) for n in (0, 1, 2, 255, 256, 257, 512, 513)]
    got = run_gpu(ctx, oracle, streams, 400, 48, with_resets)
    compare(oracle, streams, got, 400, 48, with_resets)


def test_capacity_overwrites_the_last_entry_and_scan_overflow(R, oracle, ctx):
    rng = np.random.default_rng(3)
    # scans longer than the holder (cap 50) and more scans than output slots (8)
    streams = [random_stream(oracle, rng, 4000, 0.008, 2) for _ in range(16)]
    got = run_gpu(ctx, oracle, streams, 50, 8)
    compare(oracle, streams, got, 50, 8)
    assert (got[2] > 8).any() and (got[1] == 50).any()


def test_many_scan_starts_and_many_resets_take_the_block_scan_path(R, oracle, ctx):
    rng = np.random.default_rng(23)
    streams = [random_stream(oracle, rng, 20000, 0.4, 5),       # > 4096 scan starts
               random_stream(oracle, rng, 30000, 0.01, 1500),   # > 1024 resets
               random_stream(oracle, rng, 9000, 0.45, 1100),    # exactly around both limits
               random_stream(oracle, rng, 5000, 0.002, 2)]      # list path in the same launch
    got = run_gpu(ctx, oracle, streams, 300, 64)
    compare(oracle, streams, got, 300, 64)
    assert got[2][0] > 4096


def test_edge_streams(R, oracle, ctx):
    z = lambda n: np.zeros(n, np.uint32)
    mk = lambda flags: (np.array([(i, 4 * i + 4, 7, f) for i, f in enumerate(flags)], oracle.NODE_DTYPE))
    streams = [
        (mk([]), z(0)),                              # empty stream
        (mk([2, 2, 2]), z(0)),                       # never a scan start: nothing
        (mk([1]), z(0)),                             # one open scan: not published
        (mk([1, 1, 1, 1]), z(0)),                    # one-node scans
        (mk([1, 2, 2, 1, 2, 1]), np.array([0], np.uint32)),   # reset before everything: harmless
        (mk([1, 2, 2, 1, 2, 1]), np.array([3], np.uint32)),   # reset right before a scan start: kills scan 0
        (mk([1, 2, 2, 1, 2, 1]), np.array([1, 1, 4], np.uint32)),
        (mk([1, 2, 2, 1, 2, 1]), np.array([6], np.uint32)),   # after the last node
    ]
    got = run_gpu(ctx, oracle, streams, 16, 8)
    compare(oracle, streams, got, 16, 8)
    assert list(got[2]) == [0, 0, 0, 3, 2, 1, 0, 2]


def test_decode_assemble_scan_chain_stays_on_the_device(R, oracle, ctx):
    """capsules -> rpl_decode_dense_batch_dev -> rpl_assemble_scans_dev -> rpl_scan_batch_dev with no
    host round trip, against the CPU chain decode -> assemble -> ascend -> publish."""
    import torch

    n_streams, n_caps, max_nodes, max_scans = 32, 700, 8192, 8
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    host = np.stack([make_stream(oracle, n_caps, 80.0 + s, seed=900 + s, sync_every=(250 + 7 * s) if s % 3 else None)
                     for s in range(n_streams)])
    host[5, 300, 20] ^= 0x10  # a checksum error mid-stream
    dev = torch.device("cuda")
    caps = torch.from_numpy(host).to(dev)
    ccounts = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
    nodes = torch.zeros((n_streams, n_caps * 40, 8), dtype=torch.uint8, device=dev)
    ncount = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    status = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
    offs = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
    scans = torch.zeros((n_streams, max_scans, max_nodes, 8), dtype=torch.uint8, device=dev)
    slen = torch.zeros((n_streams, max_scans), dtype=torch.int32, device=dev)
    sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    NS = n_streams * max_scans
    ranges = torch.full((NS, max_nodes), float("nan"), dtype=torch.float32, device=dev)
    intens = torch.full((NS, max_nodes), float("nan"), dtype=torch.float32, device=dev)
    beams = torch.zeros(NS, dtype=torch.int32, device=dev)
    inc = torch.zeros(NS, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_dense_batch_dev(caps.data_ptr(), ccounts.data_ptr(), n_streams, n_caps, 31, nodes.data_ptr(),
                               ncount.data_ptr(), capsule_status=status.data_ptr(),
                               capsule_node_offset=offs.data_ptr())
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.assemble_scans_dev(nodes.data_ptr(), ncount.data_ptr(), n_streams, n_caps * 40, max_nodes, max_scans,
                           max_nodes, scans.data_ptr(), slen.data_ptr(), sps.data_ptr(),
                           capsule_status=status.data_ptr(), capsule_node_offset=offs.data_ptr(),
                           capsule_counts=ccounts.data_ptr(), stride_capsules=n_caps)
    params = R.scan_params(1, 0, 0, 1)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.scan_batch_dev(scans.data_ptr(), slen.data_ptr(), NS, max_nodes, params, ranges=ranges.data_ptr(),
                       intensities=intens.data_ptr(), beam_counts=beams.data_ptr(), angle_increment=inc.data_ptr())
    ctx.synchronize()
    torch.cuda.synchronize()
    hr = ranges.cpu().numpy().reshape(n_streams, max_scans, max_nodes)
    hb = beams.cpu().numpy().reshape(n_streams, max_scans)
    hs, hl = sps.cpu().numpy(), slen.cpu().numpy()
    total = 0
    for s in range(n_streams):
        en, es, eo, _ = oracle.dense_decode(host[s], 31, 0)
        e, elen, ek = oracle.assemble_scans(en, oracle.resets_from_capsules(es, eo), max_nodes, max_scans)
        assert hs[s] == ek
        for k in range(min(ek, max_scans)):
            assert hl[s, k] == elen[k]
            rc, asc = oracle.ascend(e[k, : elen[k]].copy())
            hdr, r, _ = oracle.publish(asc, oracle.scan_params(1, 0, 0, 1, 40.0, 0.1))
            assert hb[s, k] == hdr.beam_count
            assert (hr[s, k, : hdr.beam_count].view(np.uint32) == r.view(np.uint32)).all()
            total += 1
    assert total > 2 * n_streams


@pytest.mark.parametrize("max_nodes,mode_a,emit", [(4096, 0, False), (4096, 1, True), (2000, 0, True)])
def test_scan_views_equal_the_copying_chain(R, oracle, max_nodes, mode_a, emit):
    """decode -> rpl_assemble_scan_views_dev -> rpl_scan_views_dev (revolutions read where the decoder left them)
    against decode -> rpl_assemble_scans_dev -> rpl_scan_batch_dev (revolutions copied out first): same LaserScan,
    same ascended nodes, same counts -- including revolutions longer than the holder capacity (max_nodes = 2000 <
    3200: the capacity rule is applied in place) and views that start on odd nodes."""
    import torch

    n_streams, n_caps, max_scans = 24, 640, 10
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    host = np.stack([make_stream(oracle, n_caps, 80.0 + s, seed=1900 + s, sync_every=(200 + 13 * s) if s % 4 else None)
                     for s in range(n_streams)])
    dev = torch.device("cuda")
    NS = n_streams * max_scans

    def run(view_mode):
        caps = torch.from_numpy(host).to(dev)
        ccounts = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
        nodes = torch.zeros((n_streams, n_caps * 40, 8), dtype=torch.uint8, device=dev)
        ncount = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        status = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
        offs = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
        slen = torch.zeros((n_streams, max_scans), dtype=torch.int32, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        ranges = torch.full((NS, max_nodes), float("nan"), dtype=torch.float32, device=dev)
        intens = torch.full((NS, max_nodes), float("nan"), dtype=torch.float32, device=dev)
        nodes_out = torch.zeros((NS, max_nodes, 8), dtype=torch.uint8, device=dev)
        beams = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, dtype=torch.float32, device=dev)
        st = torch.zeros(NS, dtype=torch.int32, device=dev)
        starts_stride = 8 if view_mode == 2 else 64  # 8: the list of some streams overflows (fallback to the flag pass)
        starts = torch.zeros((n_streams, starts_stride), dtype=torch.int32, device=dev)
        scnt = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
        ctx.decode_dense_batch_dev(caps.data_ptr(), ccounts.data_ptr(), n_streams, n_caps, 31, nodes.data_ptr(),
                                   ncount.data_ptr(), capsule_status=status.data_ptr(),
                                   capsule_node_offset=offs.data_ptr(),
                                   scan_starts=starts.data_ptr() if view_mode >= 2 else None, starts_stride=starts_stride,
                                   scan_start_counts=scnt.data_ptr() if view_mode >= 2 else None)
        params = R.scan_params(1, mode_a, 0, 1)
        kw = dict(ranges=ranges.data_ptr(), intensities=intens.data_ptr(), beam_counts=beams.data_ptr(),
                  angle_increment=inc.data_ptr(), status=st.data_ptr(), nodes_out=nodes_out.data_ptr() if emit else None)
        if view_mode:
            views = torch.zeros((n_streams, max_scans, 2), dtype=torch.int32, device=dev)
            if view_mode >= 2:  # the decoder's scan-start list instead of the flag pass
                torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
                ctx.assemble_scan_views_starts_dev(nodes.data_ptr(), ncount.data_ptr(), n_streams, n_caps * 40,
                                                   starts.data_ptr(), starts_stride, scnt.data_ptr(), max_nodes, max_scans,
                                                   views.data_ptr(), slen.data_ptr(), sps.data_ptr(),
                                                   capsule_status=status.data_ptr(), capsule_node_offset=offs.data_ptr(),
                                                   capsule_counts=ccounts.data_ptr(), stride_capsules=n_caps)
            else:
                torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
                ctx.assemble_scan_views_dev(nodes.data_ptr(), ncount.data_ptr(), n_streams, n_caps * 40, max_nodes, max_scans,
                                            views.data_ptr(), slen.data_ptr(), sps.data_ptr(),
                                            capsule_status=status.data_ptr(), capsule_node_offset=offs.data_ptr(),
                                            capsule_counts=ccounts.data_ptr(), stride_capsules=n_caps)
            torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
            ctx.scan_views_dev(nodes.data_ptr(), n_streams * n_caps * 40, views.data_ptr(), NS, max_nodes, params, **kw)
        else:
            scans = torch.zeros((n_streams, max_scans, max_nodes, 8), dtype=torch.uint8, device=dev)
            torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
            ctx.assemble_scans_dev(nodes.data_ptr(), ncount.data_ptr(), n_streams, n_caps * 40, max_nodes, max_scans,
                                   max_nodes, scans.data_ptr(), slen.data_ptr(), sps.data_ptr(),
                                   capsule_status=status.data_ptr(), capsule_node_offset=offs.data_ptr(),
                                   capsule_counts=ccounts.data_ptr(), stride_capsules=n_caps)
            torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
            ctx.scan_batch_dev(scans.data_ptr(), slen.data_ptr(), NS, max_nodes, params, **kw)
        ctx.synchronize()
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in (slen, sps, beams, inc, st, ranges, intens, nodes_out)]

    a = run(0)
    for b in (run(1), run(2), run(3)):
        _compare_chain_runs(a, b, NS, n_streams, max_nodes, emit)
    ctx.close()


def _compare_chain_runs(a, b, NS, n_streams, max_nodes, emit):
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all() and a[1].sum() > 2 * n_streams
    assert (a[2] == b[2]).all() and (a[3].view(np.uint32) == b[3].view(np.uint32)).all() and (a[4] == b[4]).all()
    for s in range(NS):
        m, n = int(a[2][s]), int(a[0].reshape(-1)[s])
        assert (a[5][s, :m].view(np.uint32) == b[5][s, :m].view(np.uint32)).all(), s
        assert (a[6][s, :m].view(np.uint32) == b[6][s, :m].view(np.uint32)).all(), s
        if emit:
            assert (a[7][s, :n] == b[7][s, :n]).all(), s
    if max_nodes < 3200:
        assert (a[0] == max_nodes).any()  # capped revolutions were part of the comparison


@pytest.mark.parametrize("n_streams,max_nodes", [(30, 3328), (150, 3328), (150, 4096), (90, 2048)])
def test_wire_bytes_to_laserscan_in_one_host_call(R, oracle, n_streams, max_nodes):
    """rpl_chain_dense_laserscan (host buffers, chunked over both lanes) against the CPU chain
    decode -> assemble -> ascend -> publish: one chunk / several chunks, revolutions below, at and above the
    holder capacity (3200..3440 nodes per revolution)."""
    n_caps, max_scans = 1500, 20
    ctx = R.Context(0, max_nodes, 40 * max_scans)  # 40 streams per chunk at most
    host = np.stack([make_stream(oracle, n_caps, 80.0 + (s % 7), seed=3000 + s, sync_every=(300 + 11 * (s % 5)) if s % 3 else None)
                     for s in range(n_streams)])
    counts = np.full(n_streams, n_caps, np.uint32)
    counts[7], counts[8] = 0, 123
    out = ctx.chain_dense_laserscan(host, counts, R.scan_params(1, 0, 0, 1), max_nodes, max_scans)
    total = 0
    for s in list(range(0, n_streams, 9)) + [7, 8, n_streams - 1]:
        en, es, eo, _ = oracle.dense_decode(host[s, : counts[s]], 31, 0)
        e, elen, ek = oracle.assemble_scans(en, oracle.resets_from_capsules(es, eo), max_nodes, max_scans)
        assert out["scans_per_stream"][s] == ek
        for k in range(max_scans):
            slot = s * max_scans + k
            if k >= min(ek, max_scans):
                assert out["beam_counts"][slot] == 0
                continue
            # stable tie rule on both sides: a revolution cut by the holder's capacity ends with the revolution's last
            # node, whose angle can equal that of the scan-start node (the start is flagged one sample before the wrap)
            rc, asc = oracle.ascend(e[k, : elen[k]].copy(), stable=True)
            hdr, r, it = oracle.publish(asc, oracle.scan_params(1, 0, 0, 1, 40.0, 0.1), stable=True)
            assert out["beam_counts"][slot] == hdr.beam_count, (s, k, elen[k])
            got_r = out["ranges"][slot, : hdr.beam_count].view(np.uint32)
            bad = np.nonzero(got_r != r.view(np.uint32))[0]
            if bad.size:  # diagnostics: the same revolution through the plain batch call (no views, no chain)
                one = np.zeros((1, max_nodes), R.NODE_DTYPE)
                one[0, : elen[k]] = e[k, : elen[k]].view(R.NODE_DTYPE)
                chk = R.Context(0, max_nodes, 1)
                alt = chk.scan_batch(one, np.array([elen[k]], np.uint32), R.scan_params(1, 0, 0, 1))
                chk.close()
                alt_ok = bool((alt["ranges"][0, : hdr.beam_count].view(np.uint32) == r.view(np.uint32)).all())
                where = [int(np.nonzero(got_r == v)[0][0]) if (got_r == v).any() else -1 for v in r.view(np.uint32)[bad[:4]]]
                raise AssertionError((s, k, int(elen[k]), int(hdr.beam_count), bad[:8].tolist(), int(bad.size),
                                      "plain batch call ok" if alt_ok else "plain batch call ALSO wrong",
                                      out["ranges"][slot, bad[:4]].tolist(), r[bad[:4]].tolist(), where))
            assert (out["intensities"][slot, : hdr.beam_count].view(np.uint32) == it.view(np.uint32)).all(), (s, k)
            total += 1
    assert total > 20
    ctx.close()


def test_stateful_decode_and_assembly_alternate_on_one_context(R, oracle):
    """Regression (round-1 review): stateful decodes and the assembler's reset-prefix scratch share one context.
    Three rounds of decode (0x85, state carried from round to round) -> assemble on ONE context, stream counts
    growing so that the assembler's scratch is reallocated in between, every round compared with the oracle."""
    import torch

    dev = torch.device("cuda")
    c = R.Context(0, 4096, 64)
    try:
        carried = {}
        for rnd, n_streams in enumerate((8, 40, 24)):
            n_caps = 160 + 16 * rnd
            host = np.stack([make_stream(oracle, n_caps, 30.0 + s, seed=9000 + 100 * rnd + s, sync_every=40 + s)
                             for s in range(n_streams)])
            state_h = np.zeros((n_streams, 2), np.uint32)
            for s in range(n_streams):
                state_h[s] = carried.get(s, (s & 1, 0))
            caps = torch.from_numpy(host).to(dev)
            counts = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
            state = torch.from_numpy(state_h.view(np.int32)).to(dev)
            state_out = torch.zeros((n_streams, 2), dtype=torch.int32, device=dev)
            nodes = torch.zeros((n_streams, n_caps * 40, 8), dtype=torch.uint8, device=dev)
            ncount = torch.zeros(n_streams, dtype=torch.int32, device=dev)
            status = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
            offs = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
            torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
            c.decode_capsules_batch_dev(0x85, caps.data_ptr(), counts.data_ptr(), n_streams, n_caps, 31, nodes.data_ptr(),
                                        ncount.data_ptr(), state_in=state.data_ptr(), capsule_status=status.data_ptr(),
                                        capsule_node_offset=offs.data_ptr(), state_out=state_out.data_ptr())
            max_nodes, max_scans = 700, 16
            scans = torch.zeros((n_streams, max_scans, max_nodes, 8), dtype=torch.uint8, device=dev)
            slen = torch.zeros((n_streams, max_scans), dtype=torch.int32, device=dev)
            sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
            c.assemble_scans_dev(nodes.data_ptr(), ncount.data_ptr(), n_streams, n_caps * 40, max_nodes, max_scans, max_nodes,
                                 scans.data_ptr(), slen.data_ptr(), sps.data_ptr(), capsule_status=status.data_ptr(),
                                 capsule_node_offset=offs.data_ptr(), capsule_counts=counts.data_ptr(), stride_capsules=n_caps)
            c.synchronize()
            torch.cuda.synchronize()
            hn = nodes.cpu().numpy().view(oracle.NODE_DTYPE).reshape(n_streams, n_caps * 40)
            so = state_out.cpu().numpy().astype(np.uint32)
            g = scans.cpu().numpy().view(oracle.NODE_DTYPE).reshape(n_streams, max_scans, max_nodes)
            gl, gk = slen.cpu().numpy(), sps.cpu().numpy()
            for s in range(n_streams):
                en, es, eo, est = oracle.dense_decode(host[s], 31, int(state_h[s, 0]))
                assert int(ncount[s]) == len(en), (rnd, s)
                assert (hn[s, : len(en)].view(np.uint64) == en.view(np.uint64)).all(), (rnd, s)
                assert int(so[s, 0]) == int(est), (rnd, s)
                e, elen, ek = oracle.assemble_scans(en, oracle.resets_from_capsules(es, eo), max_nodes, max_scans)
                assert int(gk[s]) == ek, (rnd, s)
                for k in range(min(ek, max_scans)):
                    assert int(gl[s, k]) == int(elen[k]) and (g[s, k, : elen[k]].view(np.uint64) == e[k, : elen[k]].view(np.uint64)).all()
                carried[s] = (int(so[s, 0]), 0)
    finally:
        c.close()
