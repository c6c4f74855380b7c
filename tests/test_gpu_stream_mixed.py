"""Mixed byte sessions (rpl_capsule_stream_create_bytes_mixed, rpl_capsule_stream_set_answer_types): one byte session
whose streams each have their own answer type, switched between pushes.

The rule for every case: stream s of the mixed session gives, bit for bit, what a one-stream create_bytes session of
its type gives when fed the same pieces with the same params -- ranges, intensities, beam counts, angle increments,
scans_per_stream, scan-begin stamps, state, counters, clouds, grabbed nodes and the bytes of both message kinds.  Across
a switch the stream is two such sessions in a row: the old type's up to the switch, then a fresh one of the new type fed
only the bytes after it, and its counters are the sum of the two.  The one-stream byte sessions are pinned against the
reference by the other stream-session tests."""
import numpy as np
import pytest

from test_capsule_bytes_pieces import raw_stream
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_lidars import FLAVOURS, MAX_NODES, MS, Drive, fleet_settings, lidar, receive_times, slots
from test_normal_stream_pieces import normal_stream

pytestmark = pytest.mark.gpu

TYPES = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
SIZES = [0, 1, 2, 97, 300, 2000, 6001, 12000]  # bytes per push: empty pushes, cuts inside frames and records
TIMING = (63, 256000, 17, 0)
CLOUD = dict(range_min=0.15, range_max=40.0, intensity_min=20.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def type_stream(O, ans, seed):
    """a damaged raw byte stream of answer type ans"""
    if ans == 0x81:
        return normal_stream(8000, seed, nodes_per_rev=2000, noise=50)
    return raw_stream(O, ans, seed, n_caps=100 if ans == 0x83 else 300)


class MixedDrive(Drive):
    """Drive's pushes on a mixed session"""

    def __init__(self, R, ctx, types, stride):
        self.R, self.kind, self.ans, self.n, self.stride, self.max_nodes = R, "bytes", 0, len(types), stride, MAX_NODES
        self.ms = MS
        self.sess = R.MixedByteStreamSession(ctx, types, stride, MAX_NODES, MS)


def one_drive(R, ctx, ans, stride):
    return Drive(R, ctx, "normal" if ans == 0x81 else "bytes", ans, 1, stride)


def state(R, sess):
    """(open_nodes, held_capsule, held_bytes) of every stream, whatever the session's type"""
    return [a.tolist() for a in R.CapsuleByteStreamSession.state(sess)]


def counters(sess):
    return [tuple(int(v) for v in row) for row in sess.counters().tolist()]


class Row:
    """stream s's oracle: one-stream create_bytes sessions in a row, a fresh one at every switch of its type"""

    def __init__(self, R, ctx, ans, stride):
        self.R, self.ctx, self.stride = R, ctx, stride
        self.before = (0,) * 14
        self.one = one_drive(R, ctx, ans, stride)

    def switch(self, ans):
        self.before = self.counters()
        self.one.close()
        self.one = one_drive(self.R, self.ctx, ans, self.stride)

    def counters(self):
        return tuple(a + b for a, b in zip(self.before, counters(self.one.sess)[0]))

    def close(self):
        self.one.close()


class Fleet:
    """a mixed session and its rows; params per stream (settings: RPL_FLAG_PER_STREAM) or uniform"""

    def __init__(self, R, ctx, types, stride, settings=None):
        self.R, self.n, self.settings = R, len(types), settings
        self.mixed = MixedDrive(R, ctx, types, stride)
        self.rows = [Row(R, ctx, t, stride) for t in types]
        if settings:
            self.mixed.sess.set_lidars([lidar(R, st) for st in settings])
            self.fp = R.scan_params(1, 1, 1, 1, R.FLAG_PER_STREAM)
            self.fcp = R.cloud_params(**CLOUD, is_new_protocol=0, flags=R.CLOUD_PER_STREAM)
        else:
            self.fp = R.scan_params(0, 1, 0, 1)
            self.fcp = R.cloud_params(**CLOUD, is_new_protocol=1)

    def one_params(self, s):
        """(scan params, cloud params, timing) of row s's sessions"""
        R = self.R
        if not self.settings:
            return self.fp, self.fcp, R.Timing(*TIMING)
        st = self.settings[s]
        return R.scan_params(st[0], st[1], st[2], 1), R.cloud_params(**CLOUD, is_new_protocol=st[0]), R.Timing(*st[3])

    def push(self, push, flavour, rx=None):
        """push into the mixed session and every row; compare everything stream by stream.  Returns scans published."""
        R = self.R
        timing = None if self.settings else R.Timing(*TIMING)
        got = self.mixed.push(push, self.fp, flavour, timing, rx)
        published = 0
        for s, row in enumerate(self.rows):
            p1, _, t1 = self.one_params(s)
            exp = row.one.push([push[s]], p1, flavour, t1, None if rx is None else rx[s:s + 1])
            assert slots(got, s) == slots(exp, 0), s
            published += int(exp["scans_per_stream"][0])
        self.check_last_push()
        return published

    def check_last_push(self):
        """state, counters, clouds, nodes and messages of every stream against its row"""
        R, sess = self.R, self.mixed.sess
        st, ct = state(R, sess), counters(sess)
        xc = sess.cloud(self.fcp)
        nodes, nst = sess.nodes(apply_ascend=True)
        fl, fc = sess.laserscan_msgs(self.fp, 1234), sess.cloud_msgs(self.fcp, 1234)
        for s, row in enumerate(self.rows):
            one = row.one.sess
            p1, c1, _ = self.one_params(s)
            assert [a[s] for a in st] == [a[0] for a in state(R, one)], s
            assert ct[s] == row.counters(), s
            oc = one.cloud(c1)
            sl = slice(s * MS, (s + 1) * MS)
            pc = xc["point_counts"][sl]
            assert pc.tolist() == oc["point_counts"].tolist(), s
            for j in range(MS):
                assert xc["xyzi"][s * MS + j, : pc[j]].tobytes() == oc["xyzi"][j, : pc[j]].tobytes(), (s, j)
            on, ost = one.nodes(apply_ascend=True)
            assert [a.tobytes() for a in nodes[sl]] == [a.tobytes() for a in on], s
            assert list(nst[sl]) == list(ost), s
            assert fl[sl] == one.laserscan_msgs(p1, 1234), s
            assert fc[sl] == one.cloud_msgs(c1, 1234), s

    def close(self):
        self.mixed.close()
        for row in self.rows:
            row.close()


def pieces_of(rng, streams):
    pieces, _ = _pieces_from_cuts(streams, [_random_cuts(rng, len(c), SIZES) for c in streams])
    return pieces, max(1, max(len(p) for push in pieces for p in push))


@pytest.mark.parametrize("per_stream", [False, True], ids=["uniform", "per_stream"])
@pytest.mark.parametrize("flavour", FLAVOURS)
def test_all_six_types_in_one_session(R, oracle, flavour, per_stream):
    """24 damaged streams cycling through 0x81..0x86, cut at random (empty pushes, cuts inside frames and records).
    The context's max_scans holds three streams' slots, so host and device pushes run in eight chunks of three types."""
    n = 24
    rng = np.random.default_rng(FLAVOURS.index(flavour) + 10 * per_stream)
    types = [TYPES[s % 6] for s in range(n)]
    streams = [type_stream(oracle, t, 9000 + s) for s, t in enumerate(types)]
    pieces, stride = pieces_of(rng, streams)
    rx = receive_times(rng, "bytes", streams, pieces, stride) if flavour.endswith("_ts") else [None] * len(pieces)
    ctx = R.Context(0, MAX_NODES, 3 * MS)
    fleet = Fleet(R, ctx, types, stride, fleet_settings(n) if per_stream else None)
    published = sum(fleet.push(push, flavour, rx[t]) for t, push in enumerate(pieces))
    assert published > 2 * n
    fleet.close()
    ctx.close()


# three phases of pushes: the types of 12 streams in each, and the masks of the two switches between them.
# Switch 1: 0 express -> 0x81, 1 0x81 -> dense, 2 HQ -> express, 3 masked with its own type (left alone), 4 dense -> HQ,
# 5 ultra-dense -> 0x81, 7 ultra -> ultra-dense; 10 is not masked and its differing entry is not taken.
# Switch 2: 0 0x81 -> express (back), 1 dense -> 0x81, 2 express -> HQ (back), 3 ultra -> dense, 4 HQ -> ultra-dense,
# 5 0x81 -> ultra, 6 express -> HQ, 9 masked with its own type, 11 HQ -> express.
PHASE_PUSHES = 6
PHASE_TYPES = [
    [0x82, 0x81, 0x83, 0x84, 0x85, 0x86, 0x82, 0x84, 0x81, 0x85, 0x86, 0x83],
    [0x81, 0x85, 0x82, 0x84, 0x83, 0x81, 0x82, 0x86, 0x84, 0x85, 0x81, 0x83],
    [0x82, 0x81, 0x83, 0x85, 0x86, 0x84, 0x83, 0x82, 0x86, 0x85, 0x82, 0x82],
]
PHASE_MASKS = [
    None,
    [1, 1, 1, 1, 1, 1, 0, 1, 0, 0, 0, 0],
    [1, 1, 1, 1, 1, 1, 1, 0, 0, 1, 0, 1],
]


def effective_types():
    """each phase's type of every stream"""
    eff = [list(PHASE_TYPES[0])]
    for k in (1, 2):
        eff.append([PHASE_TYPES[k][s] if PHASE_MASKS[k][s] else eff[-1][s] for s in range(12)])
    return eff


def switch_pieces(O, rng):
    """per push the pieces of every stream: each run of phases of one type is one stream of that type, cut short at a
    random byte (so that a switch drops a held frame or record and an open revolution) and split at random into the
    run's pushes"""
    eff = effective_types()
    per_stream = []
    for s in range(12):
        pushes, k = [], 0
        while k < 3:
            e = k
            while e + 1 < 3 and eff[e + 1][s] == eff[k][s]:
                e += 1
            data = type_stream(O, eff[k][s], 12000 + 10 * s + k)
            data = data[: len(data) - int(rng.integers(1, 200))]
            cuts = sorted(int(c) for c in rng.integers(0, len(data) + 1, (e - k + 1) * PHASE_PUSHES - 1)) + [len(data)]
            lo = 0
            for c in cuts:
                pushes.append(data[lo:c])
                lo = c
            k = e + 1
        per_stream.append(pushes)
    pieces = [[per_stream[s][t] for s in range(12)] for t in range(3 * PHASE_PUSHES)]
    return pieces, max(1, max(len(p) for push in pieces for p in push)), eff


def last_push(sess, fp, fcp):
    """everything the calls after a push read from it: clouds, grabbed nodes, both message kinds"""
    xc = sess.cloud(fcp)
    pc = xc["point_counts"].tolist()
    nodes, nst = sess.nodes(apply_ascend=True)
    return (pc, [xc["xyzi"][i, :c].tobytes() for i, c in enumerate(pc)], [a.tobytes() for a in nodes], list(nst),
            sess.laserscan_msgs(fp, 1234), sess.cloud_msgs(fcp, 1234))


@pytest.mark.parametrize("flavour", ["host_ts", "dev"])
def test_switches_between_pushes(R, oracle, flavour):
    """masked set_answer_types between pushes: capsule types to 0x81 and back, to and from HQ, to the same type.  A
    switched stream drops what it held and continues as a fresh one-stream session of its new type, its counters the
    sum of both sessions'; the others are left alone; the last push's outputs do not change"""
    rng = np.random.default_rng(31 + len(flavour))
    pieces, stride, eff = switch_pieces(oracle, rng)
    rx = receive_times(rng, "bytes", None, pieces, stride) if flavour.endswith("_ts") else [None] * len(pieces)
    ctx = R.Context(0, MAX_NODES, 4 * MS)
    fleet = Fleet(R, ctx, PHASE_TYPES[0], stride)
    sess = fleet.mixed.sess
    published, dropped = 0, 0
    for t, push in enumerate(pieces):
        k = t // PHASE_PUSHES
        if t and t % PHASE_PUSHES == 0:
            before, held = last_push(sess, fleet.fp, fleet.fcp), state(R, sess)
            sess.set_answer_types(PHASE_TYPES[k], np.array(PHASE_MASKS[k], np.uint8))
            assert sess.ans_types.tolist() == eff[k]
            assert last_push(sess, fleet.fp, fleet.fcp) == before
            after = state(R, sess)
            for s in range(12):
                if eff[k][s] != eff[k - 1][s]:
                    dropped += held[2][s] + held[0][s]
                    assert [a[s] for a in after] == [0, 0, 0], (t, s)
                    fleet.rows[s].switch(eff[k][s])
                else:
                    assert [a[s] for a in after] == [a[s] for a in held], (t, s)
            assert counters(sess) == [row.counters() for row in fleet.rows]
        published += fleet.push(push, flavour, rx[t])
    assert published > 12 and dropped > 0
    fleet.close()
    ctx.close()


def test_argument_checks(R, oracle):
    """a framed push on a mixed session, an invalid type at create and at set, set_answer_types on a single-type
    session, null arguments: RPL_RESULT_INVALID_DATA, no stream changed, the session still usable"""
    import ctypes as C

    L = R.lib()
    types = [0x81, 0x83, 0x86, 0x82]
    streams = [type_stream(oracle, t, 14000 + s) for s, t in enumerate(types)]
    pieces, stride = pieces_of(np.random.default_rng(2), streams)
    ctx = R.Context(0, MAX_NODES, 4 * MS)

    def refused(fn):
        with pytest.raises(R.RplError) as e:
            fn()
        assert e.value.code == R.RESULT_INVALID_DATA

    for bad in ([0x81, 0x80, 0x82, 0x83], [0x87] * 4, [0] * 4):
        refused(lambda: R.MixedByteStreamSession(ctx, bad, stride, MAX_NODES, MS))
    h = C.c_void_p()
    assert L.rpl_capsule_stream_create_bytes_mixed(ctx._h, None, 4, stride, MAX_NODES, MS, C.byref(h)) == \
        R.RESULT_INVALID_DATA
    fleet = Fleet(R, ctx, types, stride)
    sess = fleet.mixed.sess
    fleet.push(pieces[0], "host")
    # a framed push
    caps = np.zeros((4, 8, 84), np.uint8)
    p = R.scan_params(0, 1, 0, 1)
    out = {k: np.zeros(4 * MS * MAX_NODES, np.float32) for k in ("ranges", "intensities")}
    bc, inc, sps = np.zeros(4 * MS, np.uint32), np.zeros(4 * MS, np.float32), np.zeros(4, np.uint32)
    assert L.rpl_capsule_stream_push(sess._h, caps.ctypes.data, np.zeros(4, np.uint32).ctypes.data, 31, C.byref(p),
                                     out["ranges"].ctypes.data, out["intensities"].ctypes.data, bc.ctypes.data,
                                     inc.ctypes.data, sps.ctypes.data) == R.RESULT_INVALID_DATA
    # invalid types at set (masked or not), null types, a single-type session: nothing changes
    held = state(R, sess)
    refused(lambda: sess.set_answer_types([0x82, 0x82, 0x88, 0x82]))
    refused(lambda: sess.set_answer_types([0x82, 0x82, 0x88, 0x82], np.array([0, 0, 1, 0], np.uint8)))
    assert L.rpl_capsule_stream_set_answer_types(sess._h, None, None) == R.RESULT_INVALID_DATA
    assert L.rpl_capsule_stream_set_answer_types(None, None, None) == R.RESULT_INVALID_DATA
    same = np.array([0x82] * 4, np.uint32)
    with R.CapsuleByteStreamSession(ctx, 0x82, 4, stride, MAX_NODES, MS) as single:
        assert L.rpl_capsule_stream_set_answer_types(single._h, same.ctypes.data, None) == R.RESULT_INVALID_DATA
    # an invalid type outside the mask is not looked at
    sess.set_answer_types([0x81, 0x83, 0x86, 0x99], np.array([1, 1, 1, 0], np.uint8))
    assert sess.ans_types.tolist() == types and state(R, sess) == held
    for push in pieces[1:4]:
        fleet.push(push, "dev")
    fleet.close()
    ctx.close()
