"""Per-stream lidar settings of the stream sessions (rpl_*_stream_set_lidars, RPL_FLAG_PER_STREAM, RPL_CLOUD_PER_STREAM).

The rule for every case: each stream of a session pushed with the flag gives, bit for bit, what a one-stream session
gives when it is fed the same pieces with uniform params and timing equal to that stream's settings.  That covers
ranges, intensities, beam counts, angle increments, scans_per_stream, scan-begin stamps, the session clouds and the
bytes of the packed LaserScan and PointCloud2 messages.  The uniform session path is pinned against the reference by
the other stream-session tests."""
import itertools

import numpy as np
import pytest

from test_capsule_bytes_pieces import raw_stream
from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_dense_stream import _stream as dense_stream
from test_gpu_stream_cloud import hq_stream
from test_gpu_stream_stamps import _capsule_rx, _normal_rx, _rx_times
from test_normal_stream_pieces import normal_stream

pytestmark = pytest.mark.gpu

MAX_NODES, MS = 4096, 16
CHUNK_BYTES = 64  # receive-time pieces of the byte and 0x81 pushes
# sample duration, baud rate, linkage delay, interface (0 UART, 1 ETHERNET)
TIMINGS = [(31, 0, 0, 0), (63, 256000, 17, 0), (125, 1000000, 0, 1), (476, 115200, 250, 0), (31, 460800, 5, 1),
           (40, 0, 100, 1), (50, 256000, 0, 0), (90, 0, 33, 1)]
COMBOS = list(itertools.product((0, 1), (0, 1), (0, 1)))  # is_new_protocol, scan_processing, inverted
KINDS = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + [("bytes", 0x86), ("normal", 0x81)]
FLAVOURS = ["host", "dev", "host_ts", "dev_ts"]


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def fleet_settings(n):
    """all 8 protocol x mode x inverted combinations, each twice with different timings"""
    return [(*COMBOS[s % 8], TIMINGS[(s + 3 * (s // 8)) % len(TIMINGS)]) for s in range(n)]


def lidar(R, st):
    return R.lidar_settings(st[0], st[1], st[2], R.Timing(*st[3]))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32).tobytes()


def stream_data(O, kind, ans, n, seed0):
    """n streams of about 4.5 revolutions, and the units (capsules or bytes) of about one revolution"""
    if kind == "normal":
        return [normal_stream(14500, seed0 + s, nodes_per_rev=2900, noise=50) for s in range(n)], 5 * 2900
    if kind == "bytes":
        return [raw_stream(O, ans, seed0 + s) for s in range(n)], 40 * O.capsule_bytes(ans)
    if ans == 0x85:
        return [dense_stream(O, 360, seed0 + s, sync_every=(150 + 7 * s) if s % 3 else None) for s in range(n)], 80
    n_caps, rev = {0x82: (400, 80), 0x83: (134, 30), 0x84: (134, 30), 0x86: (200, 45)}[ans]
    return [format_stream(O, ans, n_caps, seed0 + s, sync_every=(250 + 7 * (s % 11)) if s % 3 else None,
                          near=(ans == 0x86 and s % 2 == 0)) for s in range(n)], rev


def split(rng, streams, rev):
    sizes = [0, 1, 2, rev // 3, rev, rev + 1, 2 * rev + 2]
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, len(c), sizes) for c in streams])
    return pieces, max(1, max(len(p) for push in pieces for p in push))


class Drive:
    """one session of any kind, pushed host or device, stamped or not; outputs come back as host arrays"""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes=MAX_NODES, max_scans=MS):
        self.R, self.kind, self.ans, self.n, self.stride, self.max_nodes = R, kind, ans, n, stride, max_nodes
        self.ms = max_scans
        if kind == "normal":
            self.sess = R.NormalStreamSession(ctx, n, stride, max_nodes, max_scans)
        elif kind == "bytes":
            self.sess = R.CapsuleByteStreamSession(ctx, ans, n, stride, max_nodes, max_scans)
        else:
            self.sess = R.CapsuleStreamSession(ctx, ans, n, stride, max_nodes, max_scans)

    def push(self, units, params, flavour, timing=None, rx=None):
        """units: per stream the capsules (bytes); timing: R.Timing or None; rx: the stamped push's receive times"""
        R, n, framed = self.R, self.n, self.kind == "framed"
        buf = np.zeros((n, self.stride, self.sess.capsule_bytes), np.uint8) if framed else \
            np.full((n, self.stride), 0xEE, np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(units):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        sd = {} if self.kind == "normal" else dict(sample_duration_us=timing.sample_duration_us if timing else 31)
        kw = {}
        if flavour.endswith("_ts"):
            kw = dict(rx_us=rx, timing=timing) if framed else dict(chunk_bytes=CHUNK_BYTES, chunk_rx_us=rx, timing=timing)
        if flavour.startswith("host"):
            out = self.sess.push(buf, cnt, params, **sd, **kw)
            if not kw:
                out["scan_begin_ts_us"] = None
            return out
        import torch

        dev = torch.device("cuda", 0)
        NS = n * self.ms
        d_buf, d_cnt = torch.from_numpy(buf).to(dev), torch.from_numpy(cnt.view(np.int32)).to(dev)
        r = torch.full((NS, self.max_nodes), -1.0, device=dev)
        it = torch.full((NS, self.max_nodes), -1.0, device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, dtype=torch.float32, device=dev)
        sps = torch.zeros(n, dtype=torch.int32, device=dev)
        ts = torch.full((NS,), -1, dtype=torch.int64, device=dev)
        if kw:
            d_rx = torch.from_numpy(np.ascontiguousarray(rx, np.uint64).view(np.int64)).to(dev)
            if framed:
                kw["rx_us"] = d_rx.data_ptr()
            else:
                kw["chunk_rx_us"] = d_rx.data_ptr()
            kw["scan_begin_ts_us"] = ts.data_ptr()
        torch.cuda.synchronize()
        self.sess.push_dev(d_buf.data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                           inc.data_ptr(), sps.data_ptr(), **sd, **kw)
        self.sess._ctx.synchronize()
        return dict(ranges=r.cpu().numpy(), intensities=it.cpu().numpy(), beam_counts=bc.cpu().numpy().view(np.uint32),
                    angle_increment=inc.cpu().numpy(), scans_per_stream=sps.cpu().numpy().view(np.uint32),
                    scan_begin_ts_us=ts.cpu().numpy().view(np.uint64) if kw else None)

    def close(self):
        self.sess.close()


def slots(out, s, ms=MS):
    """stream s's part of a push's outputs (ms: the session's max_scans)"""
    k = int(out["scans_per_stream"][s])
    res = [k]
    for j in range(min(k, ms)):
        i = s * ms + j
        m = int(out["beam_counts"][i])
        res.append((m, bits(out["ranges"][i, :m]), bits(out["intensities"][i, :m]), bits(out["angle_increment"][i:i + 1])))
    if out["scan_begin_ts_us"] is not None:
        res.append(out["scan_begin_ts_us"][s * ms:(s + 1) * ms].tolist())
    return res


def clouds(sess, params, s):
    out = sess.cloud(params)
    pc = out["point_counts"][s * MS:(s + 1) * MS]
    return pc.tolist(), [out["xyzi"][s * MS + j, : pc[j]].tobytes() for j in range(MS)]


def receive_times(rng, kind, streams, pieces, stride):
    """per push the receive times of every stream's units"""
    if kind == "framed":
        return _capsule_rx(pieces, [_rx_times(rng, len(c)) for c in streams], stride)
    return _normal_rx(rng, pieces, stride, CHUNK_BYTES)[0]


def run_fleet(R, ctx, kind, ans, streams, pieces, stride, flavour, settings, rng, schedule=None, cloud_kw=None,
              max_nodes=MAX_NODES, fleet_params=(1, 1, 1), check_msgs=True):
    """pushes `pieces` into one session with the flag and into one session per stream with that stream's settings as
    uniform params and timing; after every push compares outputs, clouds and messages stream by stream.  schedule:
    {push index: (new settings, mask)} applied by a masked set_lidars before that push (and by the one-stream sessions'
    params from that push on).  Returns the number of scans published."""
    n = len(streams)
    stamped = flavour.endswith("_ts")
    rx = receive_times(rng, kind, streams, pieces, stride) if stamped else [None] * len(pieces)
    fleet = Drive(R, ctx, kind, ans, n, stride, max_nodes)
    ones = [Drive(R, ctx, kind, ans, 1, stride, max_nodes) for _ in range(n)]
    table = list(settings)
    fleet.sess.set_lidars([lidar(R, st) for st in table])
    fp = R.scan_params(*fleet_params, 1, R.FLAG_PER_STREAM)
    cloud_kw = dict(range_min=0.15, range_max=40.0, intensity_min=20.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0,
                    **(cloud_kw or {}))
    flags = cloud_kw.pop("flags", 0)
    fcp = R.cloud_params(**cloud_kw, is_new_protocol=1 - fleet_params[0], flags=flags | R.CLOUD_PER_STREAM)
    published = 0
    for t, push in enumerate(pieces):
        if schedule and t in schedule:
            new, mask = schedule[t]
            fleet.sess.set_lidars([lidar(R, st) for st in new], mask)
            table = [new[s] if mask[s] else table[s] for s in range(n)]
        # a flagged stamped push may leave timing out; the flagless pushes of the one-stream sessions give theirs
        got = fleet.push(push, fp, flavour, None, rx[t])
        for s in range(n):
            st = table[s]
            one = ones[s]
            p1 = R.scan_params(st[0], st[1], st[2], 1)
            exp = one.push([push[s]], p1, flavour, R.Timing(*st[3]), None if rx[t] is None else rx[t][s:s + 1])
            assert slots(got, s) == slots(exp, 0), (t, s)
            published += int(exp["scans_per_stream"][0])
        for s in range(n):
            st, one = table[s], ones[s].sess
            assert clouds(fleet.sess, fcp, s) == clouds(one, R.cloud_params(**cloud_kw, is_new_protocol=st[0],
                                                                             flags=flags), 0), (t, s)
        if check_msgs:
            fl, fc = fleet.sess.laserscan_msgs(fp, 1234), fleet.sess.cloud_msgs(fcp, 1234)
            for s in range(n):
                st, one = table[s], ones[s].sess
                assert fl[s * MS:(s + 1) * MS] == one.laserscan_msgs(R.scan_params(st[0], st[1], st[2], 1), 1234), (t, s)
                assert fc[s * MS:(s + 1) * MS] == one.cloud_msgs(
                    R.cloud_params(**cloud_kw, is_new_protocol=st[0], flags=flags), 1234), (t, s)
    fleet.close()
    for one in ones:
        one.close()
    return published


@pytest.mark.parametrize("flavour", FLAVOURS)
@pytest.mark.parametrize("kind,ans", KINDS, ids=[f"{k}_{a:02x}" for k, a in KINDS])
def test_every_session_kind_and_push_flavour(R, oracle, kind, ans, flavour):
    """16 streams: every protocol x mode x inverted combination twice, with different timings.  The context's max_scans
    holds three streams' slots, so pushes and the cloud and message calls run in six chunks."""
    n = 16
    rng = np.random.default_rng(ans * 7 + FLAVOURS.index(flavour) + 100 * (kind == "bytes"))
    streams, rev = stream_data(oracle, kind, ans, n, 3000 + ans)
    pieces, stride = split(rng, streams, rev)
    ctx = R.Context(0, MAX_NODES, 3 * MS)
    published = run_fleet(R, ctx, kind, ans, streams, pieces, stride, flavour, fleet_settings(n), rng)
    assert published > 2 * n
    ctx.close()


@pytest.mark.parametrize("kind,ans", [("framed", 0x85), ("framed", 0x82), ("normal", 0x81), ("bytes", 0x84)])
def test_uniform_table_is_the_flagless_push(R, oracle, kind, ans):
    """the flag with every entry equal gives the bits of the push without it; the flagged push's own params and
    timing (here deliberately different) are ignored"""
    n = 12
    rng = np.random.default_rng(ans)
    streams, rev = stream_data(oracle, kind, ans, n, 5000 + ans)
    pieces, stride = split(rng, streams, rev)
    st = (1, 0, 1, (63, 256000, 17, 1))
    ctx = R.Context(0, MAX_NODES, n * MS)
    for flavour in ("host_ts", "dev"):
        rx = receive_times(rng, kind, streams, pieces, stride) if flavour == "host_ts" else [None] * len(pieces)
        a, b = Drive(R, ctx, kind, ans, n, stride), Drive(R, ctx, kind, ans, n, stride)
        a.sess.set_lidars([lidar(R, st)] * n)
        pa = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
        pb = R.scan_params(st[0], st[1], st[2], 1)
        ca = R.cloud_params(intensity_min=10.0, voxel_size=0.05, is_new_protocol=0, flags=R.CLOUD_PER_STREAM)
        cb = R.cloud_params(intensity_min=10.0, voxel_size=0.05, is_new_protocol=st[0])
        for t, push in enumerate(pieces):
            ga = a.push(push, pa, flavour, R.Timing(31, 0, 0, 0), rx[t])
            gb = b.push(push, pb, flavour, R.Timing(*st[3]), rx[t])
            for s in range(n):
                assert slots(ga, s) == slots(gb, s), (flavour, t, s)
                assert clouds(a.sess, ca, s) == clouds(b.sess, cb, s), (flavour, t, s)
            assert a.sess.laserscan_msgs(pa) == b.sess.laserscan_msgs(pb)
        a.close()
        b.close()
    ctx.close()


@pytest.mark.parametrize("ans", [0x85, 0x86])
def test_discard_threshold_per_stream(R, oracle, ans):
    """two streams of identical capsules and different sample durations: one discards an angular jump that the other
    releases, as one-stream sessions with those sample durations do"""
    O = oracle
    caps = dense_stream(O, 360, 77, sync_every=150) if ans == 0x85 else format_stream(O, ans, 200, 77, sync_every=120)
    base = O.decode_capsules(ans, caps, 31)[1] & O.CAPSULE_DISCARD
    sd = next(d for d in (20, 15, 10, 5, 2, 1) if ((O.decode_capsules(ans, caps, d)[1] & O.CAPSULE_DISCARD) != base).any())
    settings = [(1, 0, 0, (31, 0, 0, 0)), (1, 0, 0, (sd, 0, 0, 0))]
    rng = np.random.default_rng(ans)
    cuts = _random_cuts(rng, len(caps), [1, 40, 80, 161])
    pieces, _ = _pieces_from_cuts([caps, caps], [cuts, cuts])
    stride = max(len(p[0]) for p in pieces)
    ctx = R.Context(0, MAX_NODES, 2 * MS)
    fleet = Drive(R, ctx, "framed", ans, 2, stride)
    fleet.sess.set_lidars([lidar(R, st) for st in settings])
    rows = [[], []]
    for flavour in ("host", "dev_ts"):
        run_fleet(R, ctx, "framed", ans, [caps, caps], pieces, stride, flavour, settings, rng, check_msgs=False)
    for push in pieces:
        out = fleet.push(push, R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM), "host")
        for s in range(2):
            rows[s] += slots(out, s)[1:]
    assert rows[0] != rows[1]
    fleet.close()
    ctx.close()


def test_hand_off_paths_take_each_scans_mode(R, oracle):
    """duplicate-key revolutions in streams of both modes, so that the general kernel serves scans of mixed modes from
    the hand-off list; revolutions above 4096 nodes at max_nodes 8192 also hand session clouds to the general kernel"""
    O = oracle
    n = 8
    streams = [hq_stream(O, 4, (3000, 6000)[s % 2], 600 + s, dup_share=0.02) for s in range(n)]
    rng = np.random.default_rng(5)
    pieces, stride = split(rng, streams, 40)
    ctx = R.Context(0, 8192, n * MS)
    settings = [(*COMBOS[(3 * s) % 8], TIMINGS[s]) for s in range(n)]
    assert {st[1] for st in settings} == {0, 1}
    for flavour, kw in (("dev", None), ("host_ts", dict(flags=R.CLOUD_NO_FUSED))):
        published = run_fleet(R, ctx, "framed", 0x83, streams, pieces, stride, flavour, settings, rng, cloud_kw=kw,
                              max_nodes=8192, check_msgs=flavour == "dev")
        assert published > 2 * n
    ctx.close()


def test_chunks_with_modes_only_in_later_chunks(R, oracle):
    """host pushes in chunks of two streams: the first chunks are all Mode B and not inverted, the later ones carry
    Mode A, inversion, the other protocol and other timings"""
    n = 10
    rng = np.random.default_rng(11)
    streams, rev = stream_data(oracle, "framed", 0x85, n, 6100)
    pieces, stride = split(rng, streams, rev)
    settings = [(0, 0, 0, (31, 0, 0, 0))] * 6 + [(1, 1, 1, (63, 0, 5, 1)), (1, 1, 0, (125, 256000, 0, 0)),
                                                 (0, 1, 1, (31, 0, 40, 1)), (1, 0, 1, (476, 0, 0, 0))]
    ctx = R.Context(0, MAX_NODES, 2 * MS)
    for flavour in ("host_ts", "dev"):
        run_fleet(R, ctx, "framed", 0x85, streams, pieces, stride, flavour, settings, rng)
    ctx.close()


@pytest.mark.parametrize("kind,ans", [("framed", 0x82), ("normal", 0x81)])
def test_reconfigure_between_pushes(R, oracle, kind, ans):
    """a masked set_lidars between pushes flips one stream's mode and inversion and changes another stream's timing;
    the outputs follow from the next push on, like one-stream sessions whose params change at the same push"""
    n = 8
    rng = np.random.default_rng(ans + 1)
    streams, rev = stream_data(oracle, kind, ans, n, 7100 + ans)
    pieces, stride = split(rng, streams, rev)
    assert len(pieces) >= 6
    settings = fleet_settings(n)
    a, b = list(settings), list(settings)
    a[2] = (a[2][0], 1 - a[2][1], 1 - a[2][2], a[2][3])
    a[5] = (*a[5][:3], (125, 0, 77, 1 - a[5][3][3]))
    b[6] = (1 - b[6][0], *b[6][1:])
    mask_a = np.zeros(n, np.uint8)
    mask_a[[2, 5]] = 1
    mask_b = np.zeros(n, np.uint8)
    mask_b[6] = 1
    b[2] = (9, 9, 9, (1, 1, 1, 1))  # not in the mask: must not be copied
    schedule = {2: (a, mask_a), len(pieces) // 2 + 1: (b, mask_b)}
    ctx = R.Context(0, MAX_NODES, n * MS)
    for flavour in ("host_ts", "dev_ts"):
        run_fleet(R, ctx, kind, ans, streams, pieces, stride, flavour, settings, rng, schedule=schedule)
    ctx.close()


def test_argument_checks_on_the_session_handle(R, oracle):
    import ctypes as C

    O = oracle
    n = 4
    streams, rev = stream_data(O, "framed", 0x85, n, 8100)
    pieces, stride = split(np.random.default_rng(3), streams, rev)
    assert len(pieces) >= 5
    ctx = R.Context(0, MAX_NODES, n * MS)
    d = Drive(R, ctx, "framed", 0x85, n, stride)
    per = R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM)
    cpp = R.cloud_params(flags=R.CLOUD_PER_STREAM)

    def refused(fn):
        with pytest.raises(R.RplError) as e:
            fn()
        assert e.value.code == R.RESULT_INVALID_DATA

    # the flag before any set_lidars: every call that would read the table
    refused(lambda: d.push(pieces[0], per, "host"))
    refused(lambda: d.push(pieces[0], per, "dev_ts", None, receive_times(np.random.default_rng(0), "framed", streams,
                                                                          pieces, stride)[0]))
    d.push(pieces[0], R.scan_params(1, 0, 0, 1), "host")
    refused(lambda: d.sess.cloud(cpp))
    refused(lambda: d.sess.laserscan_msgs(per))
    refused(lambda: d.sess.cloud_msgs(cpp))
    # a null table, a first call that leaves a stream out, a zero sample duration: refused, the table unchanged
    assert R.lib().rpl_capsule_stream_set_lidars(d.sess._h, None, None) == R.RESULT_INVALID_DATA
    good = [(0, 0, 0, (31, 0, 0, 0)), (1, 1, 0, (63, 0, 0, 0)), (0, 1, 1, (31, 0, 9, 1)), (1, 0, 1, (90, 0, 0, 0))]
    refused(lambda: d.sess.set_lidars([lidar(R, st) for st in good], np.array([1, 1, 0, 1], np.uint8)))
    d.sess.set_lidars([lidar(R, st) for st in good])
    bad = [(1, 1, 1, (125, 0, 0, 0))] * 3 + [(1, 1, 1, (0, 0, 0, 0))]
    refused(lambda: d.sess.set_lidars([lidar(R, st) for st in bad]))
    refused(lambda: d.sess.set_lidars([lidar(R, st) for st in bad], np.array([0, 0, 0, 1], np.uint8)))
    too_long = [(1, 1, 1, (1000001, 0, 0, 0))] * n
    refused(lambda: d.sess.set_lidars([lidar(R, st) for st in too_long], np.array([1, 0, 0, 0], np.uint8)))
    ones = [Drive(R, ctx, "framed", 0x85, 1, stride) for _ in range(n)]
    for s, one in enumerate(ones):  # the history of `d`: its flagless first push
        one.push([pieces[0][s]], R.scan_params(1, 0, 0, 1), "host")
    for push in pieces[1:4]:
        got = d.push(push, per, "host")
        for s, st in enumerate(good):
            exp = ones[s].push([push[s]], R.scan_params(st[0], st[1], st[2], 1), "host", R.Timing(*st[3]))
            assert slots(got, s) == slots(exp, 0), s
    # a stamped push without the flag still needs its timing
    rx = receive_times(np.random.default_rng(1), "framed", streams, pieces, stride)[4]
    with pytest.raises(AssertionError):
        d.push(pieces[4], R.scan_params(1, 0, 0, 1), "host_ts", None, rx)
    assert R.lib().rpl_capsule_stream_push_ts(d.sess._h, None, None, None, None, C.byref(R.scan_params(1, 0, 0, 1)),
                                              None, None, None, None, None, None) == R.RESULT_INVALID_DATA
    for one in ones:
        one.close()
    d.close()
    # the non-session calls ignore both bits
    nodes = O.synth_batch(7, 6, 3000, 1)
    counts = np.full(6, 3000, np.uint32)
    for mode_a in (0, 1):
        a = ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts, R.scan_params(1, mode_a, 1, 1))
        b = ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts, R.scan_params(1, mode_a, 1, 1, R.FLAG_PER_STREAM))
        for k in ("ranges", "intensities", "beam_counts", "angle_increment"):
            assert bits(a[k]) == bits(b[k]), k
    xa, pa = ctx.cloud_batch(nodes.view(R.NODE_DTYPE), counts, R.cloud_params(intensity_min=20.0, is_new_protocol=0))
    xb, pb = ctx.cloud_batch(nodes.view(R.NODE_DTYPE), counts,
                             R.cloud_params(intensity_min=20.0, is_new_protocol=0, flags=R.CLOUD_PER_STREAM))
    assert (pa == pb).all() and bits(xa) == bits(xb)
    ctx.close()
