"""Moving live streams between stream sessions (rpl_capsule_stream_export / _import).

The definition: push P1..Pk of a stream into slot a of session A, export slot a, import the record into slot b of a
session B of the same kind and max_nodes (other n_streams, strides and max_scans, another context), push P(k+1)..Pn
into B.  A's outputs up to k followed by B's are bit for bit those of one session fed P1..Pn: LaserScans, beam counts,
angle increments, scan-begin stamps, state, every counter, session nodes and clouds, and both message kinds from the
message calls and from message pushes.  Here the stream hops between A and B after EVERY push, so one run moves it at
every push boundary, with the push flavours (host, device, stamped or not, message pushes) mixed so that either side's
last push may have been stamped or not.  The one-stream session it is compared with is pinned to the reference by the
other stream-session tests."""
import numpy as np
import pytest

from test_capsule_bytes_pieces import raw_stream
from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_byte_stream import _feature_cuts
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_fleet_scale import grids
from test_gpu_stream_lidars import Drive, bits, lidar
from test_gpu_stream_stamps import _special_cuts
from test_normal_stream_pieces import normal_stream

pytestmark = pytest.mark.gpu

MAX_NODES = 1024  # below every test stream's revolution (2000 to 3200 nodes): moves with a capped revolution open
CHUNK = 64  # receive-time pieces of the byte pushes
TIMING = (31, 256000, 17, 0)
SETTINGS = (1, 0, 1, (63, 256000, 17, 0))  # the moving stream's own lidar settings with RPL_FLAG_PER_STREAM
OTHER = (0, 1, 0, (125, 1000000, 0, 1))  # the other streams'
CLOUD = dict(range_min=0.15, range_max=40.0, intensity_min=20.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)
# the push of each step, cycled: every pair of neighbours occurs, stamped after unstamped and the reverse
FLOW = ["host_ts", "dev", "dev_ts", "host", "ls_ts", "host_ts", "cloud", "dev_ts", "ls", "host", "cloud_ts", "dev"]
KINDS = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + [("bytes", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] \
    + [("normal", 0x81)]
# (kind, ans, Mode A, per-stream settings): Mode A and B alternate, three kinds run with RPL_FLAG_PER_STREAM
CASES = [(k, a, i % 2 == 1, i in (2, 6, 10)) for i, (k, a) in enumerate(KINDS)]
HEADER, HELD = 32, 192


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


# ---- records, as include/rpl_b200.h defines them ----------------------------------------------------------------------
def record(records, offsets, i):
    """record i as a dict of its header fields, held and framer words, stamps, counters and nodes"""
    o = int(offsets[i])
    h = records[o:o + HEADER].view(np.uint32)
    kind, ans, L = int(h[2]), int(h[3]), int(h[5])
    p = o + HEADER
    held = records[p:p + HELD].view(np.uint32)
    p += HELD
    framer = None
    if kind == 1 and ans != 0x81:
        framer = records[p:p + 800].view(np.uint32)
        p += 800
    st = records[p:p + 16].view(np.uint64)
    ct = records[p + 16:p + 128].view(np.uint64)
    return dict(magic=int(h[0]), version=int(h[1]), kind=kind, ans=ans, max_nodes=int(h[4]), L=L, flags=int(h[6]),
                held=held, framer=framer, open_ts=int(st[0]), held_rx=int(st[1]), counters=ct,
                nodes=records[p + 128:p + 128 + 8 * L], size=p + 128 + 8 * L - o)


# ---- the streams --------------------------------------------------------------------------------------------------------
def stream_and_cuts(O, kind, ans, seed):
    """one stream and its cut points: around every scan-start capsule (framed), at the framing features (bytes: between
    the sync bytes, inside a frame, inside a skipped run), through records (0x81), plus random ones"""
    rng = np.random.default_rng(seed)
    if kind == "normal":
        s = normal_stream(9000, seed, nodes_per_rev=2500, noise=50)
        return s, _random_cuts(rng, len(s), [1, 2, 3, 4, 7, 800, 2501, 4000])
    if kind == "bytes":
        b = raw_stream(O, ans, seed, n_caps=90 if ans == 0x83 else 260)
        cuts = _feature_cuts(O, ans, b)
        return b, sorted(set(cuts + [len(b)]))
    caps = format_stream(O, ans, 150 if ans == 0x83 else 330, seed, sync_every=110 if ans != 0x83 else None)
    cuts = sorted(set(_special_cuts(O, ans, caps, TIMING) + _random_cuts(rng, len(caps), [1, 7, 30, 60])))
    return caps, cuts


def piece_rx(rng, kind, pieces):
    """per piece its receive times: framed, one per capsule; bytes, one per CHUNK bytes of the push"""
    t, out = 10_000_000, []
    for p in pieces:
        n = len(p) if kind == "framed" else -(-len(p) // CHUNK)
        r = t + np.cumsum(rng.integers(200, 3000, n)).astype(np.uint64)
        t = int(r[-1]) if n else t
        out.append(r)
    return out


class Sess:
    """a Drive session with the moving stream in slot `slot`; the others push nothing"""

    def __init__(self, R, ctx, kind, ans, n, slot, stride, ms, per_stream):
        self.d = Drive(R, ctx, kind, ans, n, stride, MAX_NODES, ms)
        self.R, self.kind, self.n, self.slot, self.stride, self.ms = R, kind, n, slot, stride, ms
        self.sess = self.d.sess
        if per_stream:
            self.sess.set_lidars([lidar(R, SETTINGS if s == slot else OTHER) for s in range(n)])

    def units(self, piece):
        return [piece if s == self.slot else piece[:0] for s in range(self.n)]

    def rx(self, r):
        w = self.stride if self.kind == "framed" else -(-self.stride // CHUNK)
        a = np.zeros((self.n, w), np.uint64)
        a[self.slot, :len(r)] = r
        return a

    def push(self, piece, r, flavour, prm, cprm, timing):
        """the slot's outputs of one push: (k, rows, stamps) or, for a message push, (k, messages)"""
        s, ms = self.slot, self.ms
        stamped = flavour.endswith("_ts")
        tm = timing if stamped else None
        if flavour.startswith(("ls", "cloud")):
            u = self.units(piece)
            framed = self.kind == "framed"
            buf = np.zeros((self.n, self.stride, self.sess.capsule_bytes), np.uint8) if framed else \
                np.full((self.n, self.stride), 0xEE, np.uint8)
            cnt = np.array([len(x) for x in u], np.uint32)
            buf[s, :len(piece)] = piece
            kw = dict(rx_us=self.rx(r), timing=tm, chunk_bytes=None if framed else CHUNK) if stamped else {}
            sd = timing.sample_duration_us if timing is not None else 31
            if flavour.startswith("ls"):
                msgs, sps = self.sess.push_laserscan_msgs(buf, cnt, prm, 77, sd, **kw)
            else:
                msgs, sps = self.sess.push_cloud_msgs(buf, cnt, cprm, 77, sd, **kw)
            k = int(sps[s])
            assert k <= ms
            return k, msgs[s * ms:s * ms + k]
        out = self.d.push(self.units(piece), prm, flavour, tm, self.rx(r) if stamped else None)
        k = int(out["scans_per_stream"][s])
        assert k <= ms
        rows = []
        for j in range(k):
            i = s * ms + j
            m = int(out["beam_counts"][i])
            rows.append((m, bits(out["ranges"][i, :m]), bits(out["intensities"][i, :m]),
                         bits(out["angle_increment"][i:i + 1])))
        ts = None if out["scan_begin_ts_us"] is None else out["scan_begin_ts_us"][s * ms:s * ms + k].tolist()
        return k, rows, ts

    def reads(self, prm, cprm, full):
        """the slot's state and counters and, with `full`, its nodes, clouds and both message kinds of the last push"""
        s, ms = self.slot, self.ms
        res = [[int(a[s]) for a in self.sess.state()], self.sess.counters()[s].tobytes()]
        if full:
            nodes, st = self.sess.nodes(apply_ascend=True)
            c = self.sess.cloud(cprm)
            pc = c["point_counts"][s * ms:(s + 1) * ms].tolist()
            mine = nodes[s * ms:(s + 1) * ms]
            res += [[x.tobytes() for x in mine if len(x)], [int(x) for x, y in zip(st[s * ms:(s + 1) * ms], mine) if len(y)],
                    [c["xyzi"][s * ms + j, :n].tobytes() for j, n in enumerate(pc) if n], [n for n in pc if n],
                    [m for m in self.sess.laserscan_msgs(prm, 5)[s * ms:(s + 1) * ms] if m is not None],
                    [m for m in self.sess.cloud_msgs(cprm, 5)[s * ms:(s + 1) * ms] if m is not None]]
        return res

    def close(self):
        self.d.close()


def params(R, mode_a, per_stream):
    if per_stream:
        return (R.scan_params(0, 0, 0, 1, R.FLAG_PER_STREAM), R.cloud_params(**CLOUD, flags=R.CLOUD_PER_STREAM), None)
    return (R.scan_params(1, 1 if mode_a else 0, 0, 1), R.cloud_params(**CLOUD, is_new_protocol=1), R.Timing(*TIMING))


# ---- 1, 2: the definition, a move at every push boundary ---------------------------------------------------------------
@pytest.mark.parametrize("kind,ans,mode_a,per_stream", CASES,
                         ids=[f"{k}_{a:02x}_{'A' if m else 'B'}" + ("_per_stream" if p else "") for k, a, m, p in CASES])
def test_moving_at_every_push_equals_one_session(R, oracle, kind, ans, mode_a, per_stream):
    stream, cuts = stream_and_cuts(oracle, kind, ans, 900 + ans + (7 if kind == "bytes" else 0))
    pieces = [p[0] for p in _pieces_from_cuts([stream], [cuts])[0]]
    assert len(pieces) >= 10
    rx = piece_rx(np.random.default_rng(ans), kind, pieces)
    most = max(1, max(len(p) for p in pieces))
    prm, cprm, timing = params(R, mode_a, per_stream)
    ctx_a, ctx_b = R.Context(0, MAX_NODES, 64), R.Context(0, MAX_NODES, 64)
    one = Sess(R, ctx_a, kind, ans, 1, 0, most, 9, per_stream)
    a = Sess(R, ctx_a, kind, ans, 3, 1, most + 5, 8, per_stream)
    b = Sess(R, ctx_b, kind, ans, 5, 3, 2 * most + 7, 11, per_stream)
    seen = dict(capped=False, partial=False, between=False, inside=False, skipped=False, held_rx=False)
    here, there = a, b
    for t, piece in enumerate(pieces):
        fl = FLOW[t % len(FLOW)]
        exp = one.push(piece, rx[t], fl, prm, cprm, timing)
        assert here.push(piece, rx[t], fl, prm, cprm, timing) == exp, ("push", t, fl)
        full = t % 3 == 0 or t == len(pieces) - 1
        assert here.reads(prm, cprm, full) == one.reads(prm, cprm, full), ("reads", t)
        # the move: export from here, import into there
        recs, offs = here.sess.export_streams([here.slot])
        r = record(recs, offs, 0)
        assert (r["magic"], r["version"], r["ans"], r["max_nodes"]) == (0x4D4C5052, 1, ans, MAX_NODES)
        assert r["size"] <= recs.size and recs.size % 16 == 0
        seen["capped"] |= r["L"] == MAX_NODES
        seen["partial"] |= 0 < r["L"] < MAX_NODES
        if r["framer"] is not None:
            seen["between"] |= int(r["framer"][0]) == 1
            seen["inside"] |= int(r["framer"][0]) >= 2
            seen["skipped"] |= int(r["framer"][1]) == 1
        seen["held_rx"] |= int(r["held"][43]) == 1 and bool(r["flags"] & 2)
        there.sess.import_streams([there.slot], recs, offs)
        here, there = there, here
    assert seen["capped"] and seen["partial"], seen
    if kind == "bytes":
        assert seen["inside"] and seen["between"], seen
        if ans != 0x83:
            assert seen["skipped"], seen
    if ans in (0x82, 0x84) and not per_stream:
        assert seen["held_rx"], seen
    for s in (one, a, b):
        s.close()
    ctx_a.close()
    ctx_b.close()


# ---- the other properties ------------------------------------------------------------------------------------------------
def byte_streams(O, ans, n, seed, n_caps=60):
    return [raw_stream(O, ans, seed + 11 * s, n_caps=n_caps + s % 17) for s in range(n)]


def random_pieces(streams, seed, n_push):
    rng = np.random.default_rng(seed)
    cuts = [sorted(set(rng.integers(1, len(x), n_push - 1).tolist())) + [len(x)] for x in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    return pieces, max(1, max(len(p) for push in pieces for p in push))


def chunk_rx(rng, n, stride, stamped):
    """a byte push's receive times, [n, ceil(stride / CHUNK)]"""
    if not stamped:
        return None
    w = -(-stride // CHUNK)
    return (10_000_000 + np.cumsum(rng.integers(1, 500, (n, w)), axis=1)).astype(np.uint64)


def all_reads(sess, prm, cprm):
    nodes, st = sess.nodes(apply_ascend=True)
    c = sess.cloud(cprm)
    return dict(state=[a.tolist() for a in sess.state()], counters=sess.counters(),
                nodes=[x.tobytes() for x in nodes], node_status=st.tolist(), points=c["point_counts"].tolist(),
                xyzi=[c["xyzi"][i, :n].tobytes() for i, n in enumerate(c["point_counts"].tolist())],
                ls=sess.laserscan_msgs(prm, 9), cl=sess.cloud_msgs(cprm, 9))


def stream_rows(out, s, ms):
    from test_gpu_stream_lidars import slots

    return slots(out, s, ms)


def test_export_is_a_pure_read(R, oracle):
    """a session that exports (every stream, some twice, and a size query) after every push gives what its twin that
    never exports gives, in every output"""
    n, ms = 4, 8
    streams = byte_streams(oracle, 0x84, n, 310)
    pieces, stride = random_pieces(streams, 3, 6)
    prm, cprm, timing = params(R, False, False)
    ctx = R.Context(0, MAX_NODES, 2 * n * ms)
    a, twin = Drive(R, ctx, "bytes", 0x84, n, stride, MAX_NODES, ms), Drive(R, ctx, "bytes", 0x84, n, stride, MAX_NODES, ms)
    rng = np.random.default_rng(1)
    for t, push in enumerate(pieces):
        fl = ["host_ts", "dev", "host", "dev_ts"][t % 4]
        rx = chunk_rx(rng, n, stride, fl.endswith("_ts"))
        tm = timing if rx is not None else None
        ga, gt = a.push(push, prm, fl, tm, rx), twin.push(push, prm, fl, tm, rx)
        assert [stream_rows(ga, s, ms) for s in range(n)] == [stream_rows(gt, s, ms) for s in range(n)], t
        ra = all_reads(a.sess, prm, cprm)
        a.sess.export_streams([3, 0, 3, 1, 2])
        a.sess.export_streams([])
        for k, v in all_reads(twin.sess, prm, cprm).items():
            assert (ra[k].tobytes() == v.tobytes()) if k == "counters" else ra[k] == v, (t, k)
    a.close()
    twin.close()
    ctx.close()


def test_import_disturbs_nothing_else(R, oracle):
    """B and its twin are fed the same pieces, the last one unstamped; a record goes into B's slot 2.  B's last-push
    clouds, nodes and messages (every slot), its other streams' state and counters, and its settings do not change, and
    every later push gives B's other streams what the twin gives them -- stamps included, which the unstamped push made
    unknown -- while slot 2 continues the moved stream as one session fed all of it does."""
    n, ms, slot = 4, 8, 2
    streams = byte_streams(oracle, 0x86, n, 410)
    mover = byte_streams(oracle, 0x86, 1, 777, n_caps=70)[0]
    pieces, stride = random_pieces(streams + [mover], 5, 6)
    prm, cprm, timing = R.scan_params(0, 0, 0, 1, R.FLAG_PER_STREAM), R.cloud_params(**CLOUD, flags=R.CLOUD_PER_STREAM), None
    table = [SETTINGS if s % 2 == 0 else OTHER for s in range(n)]  # slot 2: the mover's settings
    ctx = R.Context(0, MAX_NODES, 4 * n * ms)
    b, twin = Drive(R, ctx, "bytes", 0x86, n, stride, MAX_NODES, ms), Drive(R, ctx, "bytes", 0x86, n, stride, MAX_NODES, ms)
    src, one = Drive(R, ctx, "bytes", 0x86, 1, stride, MAX_NODES, ms), Drive(R, ctx, "bytes", 0x86, 1, stride, MAX_NODES, ms)
    for d, tab in ((b, table), (twin, table), (src, [SETTINGS]), (one, [SETTINGS])):
        d.sess.set_lidars([lidar(R, st) for st in tab])
    rng = np.random.default_rng(2)
    flow = ["dev_ts", "host", "host_ts", "dev", "host_ts", "dev_ts"]
    for t, push in enumerate(pieces):
        fl = flow[t]
        mfl = "host_ts" if t < 2 else fl  # the mover's pushes: stamped while in its source
        rx = chunk_rx(rng, n + 1, stride, True)
        go = one.push(push[n:], prm, mfl, None, rx[n:] if mfl.endswith("_ts") else None)
        if t < 2:
            src.push(push[n:], prm, mfl, None, rx[n:])
        ub, rb = list(push[:n]), rx[:n].copy()
        if t >= 2:
            ub[slot], rb[slot] = push[n], rx[n]
        stamped = fl.endswith("_ts")
        gb = b.push(ub, prm, fl, None, rb if stamped else None)
        gt = twin.push(push[:n], prm, fl, None, rx[:n] if stamped else None)
        others = [s for s in range(n) if t < 2 or s != slot]
        assert [stream_rows(gb, s, ms) for s in others] == [stream_rows(gt, s, ms) for s in others], t
        if t >= 2:
            assert stream_rows(gb, slot, ms) == stream_rows(go, 0, ms), t
        if t == 1:  # B's last push was unstamped: import the mover, pushed stamped so far, into slot 2
            before = all_reads(b.sess, prm, cprm)
            recs, offs = src.sess.export_streams([0])
            b.sess.import_streams([slot], recs, offs)
            after = all_reads(b.sess, prm, cprm)
            for k in ("nodes", "node_status", "points", "xyzi", "ls", "cl"):
                assert after[k] == before[k], k
            keep = [s for s in range(n) if s != slot]
            assert after["counters"][keep].tobytes() == before["counters"][keep].tobytes()
            assert after["counters"][slot].tobytes() == src.sess.counters()[0].tobytes()
            assert [[a[s] for s in keep] for a in after["state"]] == [[a[s] for s in keep] for a in before["state"]]
    for d in (b, twin, src, one):
        d.close()
    ctx.close()


def test_mixed_session_takes_the_record_type(R, oracle):
    """an 0x86 record into the slot of a mixed byte session that decodes 0x81: the slot decodes 0x86 from then on, as a
    one-stream 0x86 session fed the whole stream does, and its neighbours go on as before"""
    ms = 8
    mover = byte_streams(oracle, 0x86, 1, 515, n_caps=120)[0]
    normals = [normal_stream(3000, 60 + s, nodes_per_rev=1400, noise=50) for s in range(3)]
    pieces, stride = random_pieces([mover] + normals, 8, 5)
    prm, cprm, timing = params(R, False, False)
    ctx = R.Context(0, MAX_NODES, 16 * ms)
    mixed = R.MixedByteStreamSession(ctx, [0x81, 0x81, 0x81], stride, MAX_NODES, ms)
    src = Drive(R, ctx, "bytes", 0x86, 1, stride, MAX_NODES, ms)
    one = Drive(R, ctx, "bytes", 0x86, 1, stride, MAX_NODES, ms)
    n81 = Drive(R, ctx, "normal", 0x81, 1, stride, MAX_NODES, ms)
    rng = np.random.default_rng(4)
    for t, push in enumerate(pieces):
        stamped = t % 2 == 0
        rx = chunk_rx(rng, 4, stride, stamped)
        # slot 0 decodes 0x81 bytes up to the move and the mover from then on; slots 1 and 2 their own 0x81 streams
        u = [push[3] if t < 2 else push[0], push[1], push[2]]
        kw = {}
        if stamped:
            kw = dict(chunk_bytes=CHUNK, chunk_rx_us=np.vstack([rx[3] if t < 2 else rx[0], rx[1], rx[2]]), timing=timing)
        buf = np.full((3, stride), 0xEE, np.uint8)
        for s, p in enumerate(u):
            buf[s, :len(p)] = p
        got = mixed.push(buf, [len(p) for p in u], prm, 31, **kw)
        e1 = one.push([push[0]], prm, "host_ts" if stamped else "host", timing if stamped else None,
                      rx[:1] if stamped else None)
        if t < 2:
            src.push([push[0]], prm, "host_ts" if stamped else "host", timing if stamped else None,
                     rx[:1] if stamped else None)
        e2 = n81.push([push[1]], prm, "host_ts" if stamped else "host", timing if stamped else None,
                      rx[1:2] if stamped else None)
        if not stamped:
            got["scan_begin_ts_us"] = None
        if t >= 2:
            assert stream_rows(got, 0, ms) == stream_rows(e1, 0, ms), t
        assert stream_rows(got, 1, ms) == stream_rows(e2, 0, ms), t
        if t == 1:
            assert mixed.ans_types[0] == 0x81
            recs, offs = src.sess.export_streams([0])
            mixed.import_streams([0], recs, offs)
            assert mixed.ans_types.tolist() == [0x86, 0x81, 0x81]
            assert mixed.counters()[0].tobytes() == src.sess.counters()[0].tobytes()
    mixed.close()
    for d in (src, one, n81):
        d.close()
    ctx.close()


def test_fleet_moves_in_one_call(R, oracle):
    """2 * G8 + 37 streams exported in one call and imported in one call onto a random permutation of a larger
    session's slots: both kernels walk their grid-stride loops; every stream then continues in B as in A"""
    import torch

    _, g8, _ = grids(torch.cuda.get_device_properties(0).multi_processor_count)
    n, ms = 2 * g8 + 37, 4
    streams = [raw_stream(oracle, 0x82, 5000 + 3 * s, n_caps=30 + s % 13) for s in range(n)]
    pieces, stride = random_pieces(streams, 11, 4)
    prm, cprm, timing = params(R, False, False)
    ctx = R.Context(0, MAX_NODES, (2 * n + 5) * ms)
    a = Drive(R, ctx, "bytes", 0x82, n, stride, MAX_NODES, ms)
    b = Drive(R, ctx, "bytes", 0x82, n + 5, stride + 3, MAX_NODES, ms)
    perm = np.random.default_rng(6).permutation(n + 5)[:n]
    rng = np.random.default_rng(7)
    for t, push in enumerate(pieces):
        rx = chunk_rx(rng, n, stride, True)
        ga = a.push(push, prm, "dev_ts", timing, rx)
        if t >= 2:
            ub = [np.zeros(0, np.uint8)] * (n + 5)
            rb = np.zeros((n + 5, -(-(stride + 3) // CHUNK)), np.uint64)
            for s in range(n):
                ub[perm[s]] = push[s]
                rb[perm[s], :rx.shape[1]] = rx[s]
            gb = b.push(ub, prm, "host_ts", timing, rb)
            for s in range(n):
                assert stream_rows(gb, perm[s], ms) == stream_rows(ga, s, ms), (t, s)
            assert b.sess.counters()[perm].tobytes() == a.sess.counters().tobytes()
            assert [x[perm].tolist() for x in b.sess.state()] == [x.tolist() for x in a.sess.state()]
        if t == 1:
            recs, offs = a.sess.export_streams(np.arange(n))
            assert len(offs) == n and all(record(recs, offs, i)["ans"] == 0x82 for i in range(0, n, 97))
            b.sess.import_streams(perm, recs, offs)
    a.close()
    b.close()
    ctx.close()


INVALID = 0x80008000


def test_rejections_leave_the_session_unchanged(R, oracle):
    """every malformed record or call returns RPL_RESULT_INVALID_DATA and changes nothing: state, counters and the
    outputs of the next push are those of a twin that never saw it.  A short capacity returns
    RPL_RESULT_INSUFFICIENT_MEMORY with the right total and writes no record."""
    import ctypes as C

    from rplidar_ros2_driver_b200.capi import _p

    n, ms = 3, 8
    streams = byte_streams(oracle, 0x82, n, 620)
    pieces, stride = random_pieces(streams, 9, 4)
    prm, cprm, timing = params(R, False, False)
    ctx = R.Context(0, MAX_NODES, 8 * n * ms)
    src = Drive(R, ctx, "bytes", 0x82, n, stride, MAX_NODES, ms)
    b, twin = Drive(R, ctx, "bytes", 0x82, n, stride, MAX_NODES, ms), Drive(R, ctx, "bytes", 0x82, n, stride, MAX_NODES, ms)
    framed = R.CapsuleStreamSession(ctx, 0x82, n, 8, MAX_NODES, ms)
    other = Drive(R, ctx, "bytes", 0x82, n, stride, MAX_NODES - 2, ms)
    for d in (src, b, twin):
        for push in pieces[:2]:
            d.push(push, prm, "host", None, None)
    recs, offs = src.sess.export_streams([0, 1])
    total = recs.size
    # a short capacity: nothing written, the total reported
    buf = np.full(total, 0xCD, np.uint8)
    got_offs, got_total = np.zeros(2, np.uint64), np.zeros(1, np.uint64)
    sel = np.array([0, 1], np.uint32)
    rc = src.sess._fn("export")(src.sess._h, _p(sel), 2, _p(buf), total - 1, _p(got_offs), _p(got_total))
    assert rc == 0x80008006 and int(got_total[0]) == total and got_offs.tolist() == offs.tolist()
    assert (buf == 0xCD).all()
    r0 = record(recs, offs, 0)
    o0 = int(offs[0])

    def mutated(word=None, value=None, at=None):
        r = recs.copy()
        if word is not None:
            r[o0 + 4 * word:o0 + 4 * word + 4] = np.array([value], np.uint32).view(np.uint8)
        if at is not None:
            r[o0 + at:o0 + at + 4] = np.array([value], np.uint32).view(np.uint8)
        return r

    framer_at = HEADER + HELD
    bad = [
        ("magic", [1], mutated(0, 0x4D4C5053), offs, total),
        ("version", [1], mutated(1, 2), offs, total),
        ("kind", [1], mutated(2, 0), offs, total),
        ("answer type", [1], mutated(3, 0x84), offs, total),
        ("max_nodes", [1], mutated(4, MAX_NODES - 2), offs, total),
        ("open length", [1], mutated(5, MAX_NODES + 1), offs, total),
        ("flags", [1], mutated(6, 4), offs, total),
        ("framer position", [1], mutated(at=framer_at, value=84), offs, total),
        ("outside", [1, 2], recs, offs, total - 16),
        ("offset", [1], recs, np.array([8], np.uint64), total),
        ("duplicate", [1, 1], recs, offs, total),
        ("out of range", [n], recs, offs, total),
    ]
    assert r0["framer"] is not None
    st0, ct0 = b.sess.state(), b.sess.counters()
    for name, dst, r, o, tot in bad:
        d = np.array(dst, np.uint32)
        rc = b.sess._fn("import")(b.sess._h, _p(d), d.size, _p(r), _p(np.ascontiguousarray(o[:d.size], np.uint64)), tot)
        assert rc == INVALID, name
    d = np.array([1], np.uint32)
    assert b.sess._fn("import")(b.sess._h, _p(d), 1, None, _p(offs), total) == INVALID
    assert b.sess._fn("import")(b.sess._h, None, 1, _p(recs), _p(offs), total) == INVALID
    assert b.sess._fn("import")(b.sess._h, _p(d), 1, _p(recs), None, total) == INVALID
    for s in (framed, other.sess):  # another kind, another max_nodes
        with pytest.raises(R.RplError) as e:
            s.import_streams([1], recs[:int(offs[1])], offs[:1])
        assert e.value.code == INVALID
    # 0x81: the byte machine's state out of 0..4
    nsrc = Drive(R, ctx, "normal", 0x81, 1, 64, MAX_NODES, ms)
    nsrc.push([normal_stream(40, 5)[:33]], prm, "host", None, None)
    nrec, noff = nsrc.sess.export_streams([0])
    nrec[HEADER + 4 * 43:HEADER + 4 * 43 + 4] = np.array([5], np.uint32).view(np.uint8)
    with pytest.raises(R.RplError) as e:
        nsrc.sess.import_streams([0], nrec, noff)
    assert e.value.code == INVALID
    st1, ct1 = b.sess.state(), b.sess.counters()
    assert [a.tolist() for a in st1] == [a.tolist() for a in st0] and ct1.tobytes() == ct0.tobytes()
    for push in pieces[2:]:
        gb, gt = b.push(push, prm, "host", None, None), twin.push(push, prm, "host", None, None)
        assert [stream_rows(gb, s, ms) for s in range(n)] == [stream_rows(gt, s, ms) for s in range(n)]
        assert all_reads(b.sess, prm, cprm)["ls"] == all_reads(twin.sess, prm, cprm)["ls"]
    for d in (src, b, twin, other, nsrc):
        d.close()
    framed.close()
    ctx.close()


def test_move_across_devices(R, oracle):
    """a stream moved from a session on GPU 0 to one on GPU 1 continues as one session fed all of it"""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    ms = 8
    stream = byte_streams(oracle, 0x85, 1, 880, n_caps=200)[0]
    pieces, stride = random_pieces([stream], 12, 6)
    prm, cprm, timing = params(R, True, False)
    c0, c1 = R.Context(0, MAX_NODES, 4 * ms), R.Context(1, MAX_NODES, 4 * ms)
    one, a = Drive(R, c0, "bytes", 0x85, 1, stride, MAX_NODES, ms), Drive(R, c0, "bytes", 0x85, 2, stride, MAX_NODES, ms)
    b = R.CapsuleByteStreamSession(c1, 0x85, 3, stride + 9, MAX_NODES, ms)
    rng = np.random.default_rng(13)
    for t, push in enumerate(pieces):
        rx = chunk_rx(rng, 1, stride, True)
        e = one.push(push, prm, "host_ts", timing, rx)
        if t < 3:
            g = a.push([push[0], push[0][:0]], prm, "host_ts", timing, np.vstack([rx, rx]))
            assert stream_rows(g, 0, ms) == stream_rows(e, 0, ms), t
        else:
            buf = np.full((3, stride + 9), 0xEE, np.uint8)
            buf[2, :len(push[0])] = push[0]
            rb = np.zeros((3, -(-(stride + 9) // CHUNK)), np.uint64)
            rb[2, :rx.shape[1]] = rx[0]
            g = b.push(buf, [0, 0, len(push[0])], prm, 31, chunk_bytes=CHUNK, chunk_rx_us=rb, timing=timing)
            assert stream_rows(g, 2, ms) == stream_rows(e, 0, ms), t
        if t == 2:
            recs, offs = a.sess.export_streams([0])
            b.import_streams([2], recs, offs)
    one.close()
    a.close()
    b.close()
    c0.close()
    c1.close()
