"""The stream sessions at fleet scale: more streams than CTAs in every per-stream session kernel, and slot tables past
one 1024-slot tile and one 65535-row grid.

Every per-stream session kernel walks its streams with a grid-stride loop over a capped grid: the framer and the
capsule decoders num_sms * 8 CTAs (dense num_sms * 4), the assembler num_sms * 4, the node gather num_sms * 8.  A CTA
that serves stream i, then i + grid, ... must reset its shared and register state before each stream.  The fleets here
have n = 2 * G8 + 37 streams (G8 = 8 * num_sms, G4 = 4 * num_sms) in one chunk, so every framer and decoder CTA serves
two or three streams and every assembler CTA four or five; no two streams one CTA serves are alike, and some follow a
stream whose push is empty.

The rule for every session case: the fleet session gives, bit for bit and stream by stream, what sessions of at most 64
streams give when fed the same pieces with the same params, timing and receive times (in those every CTA serves one
stream, the path the other stream-session tests pin to the oracle): LaserScans, stamps, state, counters, clouds, grabbed
nodes and both message kinds.  Streams served second and third by a CTA are also held to the whole-stream oracle.

The message table (msg_table_kernel) and the node directory (node_directory_kernel) are one CTA that carries a prefix
sum from one 1024-slot tile to the next, and the message writers split their slots into grid rows of 65535: a session
of more than 65535 slots checks every slot's offset, size and bytes.  The stateless timestamp and CDR launchers that
split at 65535 rows are checked on every stream past that.

Which kernels a push runs, and with how many CTAs, is read from the CUDA profiler's trace in a child process."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import cdr_oracle as cdr
from test_capsule_bytes_pieces import raw_stream
from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_byte_stream import _check_oracle as bytes_oracle
from test_gpu_capsule_stream import _check_oracle as framed_oracle
from test_gpu_capsule_stream import _pieces_from_cuts
from test_gpu_decode_layout import standard_records
from test_gpu_dense_stream import _check_oracle as dense_oracle
from test_gpu_dense_stream import _stream as dense_stream
from test_gpu_normal_stream import _check_oracle as normal_oracle
from test_gpu_stream_lidars import Drive, fleet_settings, lidar, receive_times, slots
from test_gpu_stream_msgs import check_packed, dev_msgs
from test_gpu_stream_nodes import check_packing, dev_nodes
from test_normal_stream_pieces import normal_stream
from test_stream_msgs_pieces import expected_cloud, expected_laserscan, pack
from test_timestamps_vs_ref import rx_times

gpu = pytest.mark.gpu

PARAMS = (1, 0, 0, 1)  # the oracle checks' params: new protocol, Mode B, not inverted, ascended
TIMING = (31, 256000, 17, 0)  # the stamped pushes' (sample duration 31 us, as the oracle checks decode)
MAX_NODES, MS = 4096, 4
SMALL = 64  # streams per reference session
HOST_CHUNK_BYTES = 16 << 20  # a host push's input per chunk (rpl_capsule_stream create)
CB = {0x81: 1, 0x82: 84, 0x83: 781, 0x84: 132, 0x85: 84, 0x86: 170}  # bytes per unit of a push (0x81: byte)
SLAB = 65535  # grid rows per launch of the message writers and the stateless timestamp and CDR launchers
CLOUD = dict(range_min=0.15, range_max=40.0, intensity_min=20.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def grids(num_sms):
    """(G4, G8, n): the assembler's and the decoders' grid caps, and the fleet size"""
    return 4 * num_sms, 8 * num_sms, 16 * num_sms + 37


@pytest.fixture(scope="module")
def sizes():
    import torch

    return grids(torch.cuda.get_device_properties(0).multi_processor_count)


def chunks(n, ctx_max_scans, max_scans, in_stream):
    """(chunk_dev, chunk_host): streams per device-push launch and per host-push chunk, as the session computes them"""
    dev = min(n, ctx_max_scans // max_scans)
    return dev, min(dev, max(1, HOST_CHUNK_BYTES // in_stream))


def unit_budget(kind, ans, n):
    """the most units (bytes, or capsules of a framed session) one stream may push so that a host chunk holds n"""
    return HOST_CHUNK_BYTES // n // (CB[ans] if kind == "framed" else 1)


# ---- the fleet's streams ---------------------------------------------------------------------------------------------
def fleet_stream(O, kind, ans, s):
    """stream s of a fleet: lengths, damage and scan-start capsules differ from stream to stream"""
    if kind == "normal":
        return normal_stream(2600 + 13 * (s % 37), 40000 + s, nodes_per_rev=1000 + 9 * (s % 53), noise=50)
    if kind == "bytes":
        n_caps = {0x82: 190, 0x83: 64, 0x84: 80, 0x85: 190, 0x86: 110}[ans] + s % 23
        return raw_stream(O, ans, 50000 + 7 * s + ans, n_caps=n_caps)
    n_caps = {0x82: 200, 0x83: 64, 0x84: 80, 0x85: 200, 0x86: 112}[ans] + s % 29
    if ans == 0x85:
        return dense_stream(O, n_caps, 60000 + s, sync_every=(150 + 7 * (s % 13)) if s % 3 else None)
    return format_stream(O, ans, n_caps, 60000 + 5 * s + ans, sync_every=(100 + 7 * (s % 11)) if s % 3 else None,
                         near=(ans == 0x86 and s % 2 == 0))


def fleet_cuts(rng, lengths, budget):
    """each stream's cut points: pieces of budget/4..budget units, about one in eight empty; every fifth stream's first
    push is empty, so that a CTA's next stream follows one that pushed nothing"""
    cuts = []
    for s, n in enumerate(lengths):
        c, at = ([0] if s % 5 == 2 else []), 0
        while at < n:
            at = at if rng.random() < 0.125 else min(n, at + int(rng.integers(budget // 4, budget + 1)))
            c.append(at)
        cuts.append(c)
    return cuts


def fleet_pieces(O, kind, ans, n, seed):
    """(streams, pieces per push, stride)"""
    streams = [fleet_stream(O, kind, ans, s) for s in range(n)]
    rng = np.random.default_rng(seed)
    pieces, _ = _pieces_from_cuts(streams, fleet_cuts(rng, [len(x) for x in streams], unit_budget(kind, ans, n)))
    return streams, pieces, max(1, max(len(p) for push in pieces for p in push))


def check_mates_differ(streams, pieces, g4, g8):
    """streams s, s + G4, s + 2 * G4, ... (one assembler CTA's, and so one framer or decoder CTA's too) differ in their
    bytes and in their cut points; some push has a stream with no units whose next stream in a CTA of either grid has"""
    n = len(streams)
    whole = [np.ascontiguousarray(x).tobytes() for x in streams]
    cut = [tuple(len(push[s]) for push in pieces) for s in range(n)]
    for s in range(g4):
        mates = range(s, n, g4)
        assert len({whole[m] for m in mates}) == len(mates), s
        assert len({cut[m] for m in mates}) == len(mates), s
    for g in (g4, g8):
        assert any(len(push[s]) == 0 < len(push[s + g]) for push in pieces for s in range(n - g)), g


# ---- a fleet session and its reference sessions ----------------------------------------------------------------------
class Fleet:
    """one session of n streams and the sessions of at most SMALL streams that hold the same streams"""

    def __init__(self, R, ctx, kind, ans, n, stride, settings=None):
        self.R, self.kind, self.n = R, kind, n
        self.big = Drive(R, ctx, kind, ans, n, stride, MAX_NODES, MS)
        self.blocks = [(lo, Drive(R, ctx, kind, ans, min(SMALL, n - lo), stride, MAX_NODES, MS))
                       for lo in range(0, n, SMALL)]
        if settings:
            self.big.sess.set_lidars([lidar(R, st) for st in settings])
            for lo, d in self.blocks:
                d.sess.set_lidars([lidar(R, st) for st in settings[lo:lo + d.n]])
            self.prm = R.scan_params(*PARAMS[:3], 1, R.FLAG_PER_STREAM)
            self.cprm = R.cloud_params(**CLOUD, flags=R.CLOUD_PER_STREAM)
            self.timing = None
        else:
            self.prm = R.scan_params(*PARAMS)
            self.cprm = R.cloud_params(**CLOUD, is_new_protocol=PARAMS[0])
            self.timing = R.Timing(*TIMING)
        self.got = [[] for _ in range(n)]  # every published row of every stream, for the oracle checks
        self.overflow = np.zeros(n, bool)  # a push published more scans than the slots

    def push(self, push, flavour, rx):
        got = self.big.push(push, self.prm, flavour, self.timing, rx)
        for lo, d in self.blocks:
            exp = d.push(push[lo:lo + d.n], self.prm, flavour, self.timing, None if rx is None else rx[lo:lo + d.n])
            for j in range(d.n):
                row = slots(got, lo + j, MS)
                assert row == slots(exp, j, MS), ("push", lo + j)
                self.got[lo + j] += [r for r in row[1:1 + min(row[0], MS)]]
                self.overflow[lo + j] |= row[0] > MS
        return int(got["scans_per_stream"].sum())

    def check_reads(self):
        """state, counters, clouds, grabbed nodes (host and device) and both message kinds of the last push"""
        import torch

        big = self.big.sess
        st, ct = big.state(), big.counters()
        xc = big.cloud(self.cprm)
        nodes, nst = big.nodes(apply_ascend=True)
        dn = dev_nodes(torch, big)
        check_packing(dn, self.n * MS)
        fl, fc = big.laserscan_msgs(self.prm, 1234), big.cloud_msgs(self.cprm, 1234)
        for lo, d in self.blocks:
            one, m = d.sess, d.n
            sl = slice(lo * MS, (lo + m) * MS)
            assert [a[lo:lo + m].tolist() for a in st] == [a.tolist() for a in one.state()], ("state", lo)
            assert ct[lo:lo + m].tobytes() == one.counters().tobytes(), ("counters", lo)
            oc = one.cloud(self.cprm)
            pc = xc["point_counts"][sl]
            assert pc.tolist() == oc["point_counts"].tolist(), ("cloud", lo)
            for i, c in enumerate(pc.tolist()):
                assert xc["xyzi"][lo * MS + i, :c].tobytes() == oc["xyzi"][i, :c].tobytes(), ("cloud", lo * MS + i)
            on, ost = one.nodes(apply_ascend=True)
            assert [a.tobytes() for a in nodes[sl]] == [a.tobytes() for a in on], ("nodes", lo)
            assert list(nst[sl]) == list(ost), ("nodes", lo)
            for i in range(sl.start, sl.stop):
                o, c = int(dn["node_offsets"][i]), int(dn["node_counts"][i])
                assert dn["nodes"][o:o + c].tobytes() == nodes[i].tobytes() and dn["status"][i] == nst[i], ("nodes_dev", i)
            assert fl[sl] == one.laserscan_msgs(self.prm, 1234), ("laserscan_msgs", lo)
            assert fc[sl] == one.cloud_msgs(self.cprm, 1234), ("cloud_msgs", lo)

    def close(self):
        self.big.close()
        for _, d in self.blocks:
            d.close()


def oracle_sample(n, g4, g8, overflow):
    """streams served first, second and third by a decoder CTA and fourth or fifth by an assembler CTA"""
    want = [3, 4 + g8, 5 + 2 * g8, 6 + 3 * g4, 7 + 4 * g4, 8 + g4, n - 1, n - 2 - g8]
    return [s for s in want if 0 <= s < n and not overflow[s]]


def check_oracle(O, kind, ans, fleet, streams, which):
    if kind == "normal":
        normal_oracle(O, fleet.got, streams, MAX_NODES, which)
    elif kind == "bytes":
        bytes_oracle(O, ans, fleet.got, streams, which)
    elif ans == 0x85:
        dense_oracle(O, fleet.got, streams, MAX_NODES, which)
    else:
        framed_oracle(O, ans, fleet.got, streams, MAX_NODES, which)


KINDS = [("bytes", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + [("normal", 0x81)] + \
        [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)]
# every kind once unstamped and once stamped (host and device pushes alternating over the kinds), the 0x82 byte session
# in all four flavours, and one run with per-stream settings
CASES = [(k, a, f, False) for i, (k, a) in enumerate(KINDS)
         for f in (("host", "dev", "host_ts", "dev_ts") if (k, a) == ("bytes", 0x82) else
                   (("host", "dev_ts") if i % 2 else ("dev", "host_ts")))] + [("bytes", 0x86, "dev_ts", True)]


def test_cases_cover_every_kind_and_flavour():
    """every kind one unstamped and one stamped flavour; all four on the 0x82 byte session; one per-stream run"""
    for k, a in KINDS:
        fl = {c[2] for c in CASES if c[:2] == (k, a) and not c[3]}
        assert fl & {"host", "dev"} and fl & {"host_ts", "dev_ts"}, (k, a)
    assert {c[2] for c in CASES if c[:2] == ("bytes", 0x82)} == {"host", "dev", "host_ts", "dev_ts"}
    assert sum(c[3] for c in CASES) == 1


def test_chunk_rule_and_budget():
    """the unit budget keeps a host chunk at the whole fleet for every kind and for SM counts around the H100's"""
    for num_sms in (114, 132, 144):
        _, _, n = grids(num_sms)
        for kind, ans in KINDS:
            in_stream = unit_budget(kind, ans, n) * (CB[ans] if kind == "framed" else 1)
            assert chunks(n, n * MS, MS, in_stream) == (n, n)
            assert chunks(n, n * MS, MS, in_stream + HOST_CHUNK_BYTES // n)[1] < n
    assert chunks(2149, 700 * 32, 32, 5000) == (700, 700)


@pytest.mark.parametrize("kind,ans", KINDS, ids=[f"{k}_{a:02x}" for k, a in KINDS])
def test_fleet_streams_differ_within_every_cta(oracle, kind, ans):
    """the case builder on the H100's 132 SMs: mates differ, some follow an empty push, every piece fits the budget"""
    g4, g8, n = grids(132)
    streams, pieces, stride = fleet_pieces(oracle, kind, ans, n, 1)
    check_mates_differ(streams, pieces, g4, g8)
    assert stride <= unit_budget(kind, ans, n) and len(pieces) >= 3


@gpu
@pytest.mark.parametrize("kind,ans,flavour,per_stream", CASES,
                         ids=[f"{k}_{a:02x}_{f}" + ("_per_stream" if p else "") for k, a, f, p in CASES])
def test_fleet_equals_small_sessions(R, oracle, sizes, kind, ans, flavour, per_stream):
    g4, g8, n = sizes
    streams, pieces, stride = fleet_pieces(oracle, kind, ans, n, KINDS.index((kind, ans)))
    check_mates_differ(streams, pieces, g4, g8)
    rng = np.random.default_rng(7 + len(flavour))
    rx = receive_times(rng, kind, streams, pieces, stride) if flavour.endswith("_ts") else [None] * len(pieces)
    ctx = R.Context(0, MAX_NODES, n * MS)
    fleet = Fleet(R, ctx, kind, ans, n, stride, fleet_settings(n) if per_stream else None)
    in_stream = stride * fleet.big.sess.capsule_bytes if kind == "framed" else stride
    assert chunks(n, n * MS, MS, in_stream) == (n, n)
    published = 0
    for t, push in enumerate(pieces):
        published += fleet.push(push, flavour, rx[t])
        if t == 1:
            fleet.check_reads()
    fleet.check_reads()
    assert published > n // 4
    if not per_stream:
        which = oracle_sample(n, g4, g8, fleet.overflow)
        assert any(s >= g8 for s in which) and any(s >= 2 * g8 for s in which), which
        check_oracle(oracle, kind, ans, fleet, streams, which)
    fleet.close()
    ctx.close()


# ---- a mixed byte session with two long type lists ---------------------------------------------------------------------
def mixed_types(n, g8):
    """0x82 and 0x84 on more than G8 streams each, two of every other type"""
    types = [0x82 if s % 2 == 0 else 0x84 for s in range(n)]
    for i, t in enumerate((0x81, 0x83, 0x85, 0x86) * 2):
        types[11 + 97 * i] = t
    assert types.count(0x82) > g8 and types.count(0x84) > g8
    return types


def mixed_stream(O, ans, s, k):
    """stream s's bytes of answer type ans in phase k"""
    if ans == 0x81:
        return normal_stream(2400 + 11 * (s % 7), 70000 + 2 * s + k, nodes_per_rev=1100, noise=50)
    return raw_stream(O, ans, 80000 + 13 * s + 3 * k + ans, n_caps={0x82: 150, 0x83: 40, 0x84: 64, 0x85: 150,
                                                                   0x86: 90}[ans] + s % 17)


class Blocks:
    """reference byte sessions of at most SMALL streams of one type each: block[s] = (drive, index)"""

    def __init__(self, R, ctx, types, members, stride):
        self.drives, self.at = [], {}
        for t in sorted({types[s] for s in members}):
            of = [s for s in members if types[s] == t]
            for lo in range(0, len(of), SMALL):
                part = of[lo:lo + SMALL]
                d = Drive(R, ctx, "normal" if t == 0x81 else "bytes", t, len(part), stride, MAX_NODES, MS)
                self.drives.append((d, part))
                for j, s in enumerate(part):
                    self.at[s] = (d, j)

    def push(self, push, prm, flavour, timing, rx, blank):
        """per stream the outputs of its block; blank: streams fed nothing (switched away from their block)"""
        res = {}
        for d, part in self.drives:
            sub = [push[s][:0] if s in blank else push[s] for s in part]
            out = d.push(sub, prm, flavour, timing, None if rx is None else rx[part])
            for j, s in enumerate(part):
                res[s] = slots(out, j, MS)
        return res

    def close(self):
        for d, _ in self.drives:
            d.close()


@gpu
def test_mixed_fleet_with_long_type_lists_and_a_switch(R, oracle, sizes):
    """a mixed byte session of n streams whose 0x82 and 0x84 lists are each longer than the framer's and decoders'
    grids; after three pushes set_answer_types moves several hundred streams between the two lists (and two 0x85 to
    0x81), and the pushes after it follow fresh sessions of the new types fed only the bytes after the switch, with
    the counters of both"""
    import test_gpu_stream_mixed as M

    g4, g8, n = sizes
    O = oracle
    types = mixed_types(n, g8)
    moved = [s for s in range(n) if types[s] in (0x82, 0x84) and s % 7 in (1, 4)][:400] + \
        [s for s in range(n) if types[s] == 0x85]
    new = list(types)
    for s in moved:
        new[s] = {0x82: 0x84, 0x84: 0x82, 0x85: 0x81}[types[s]]
    assert len(moved) >= 300
    rng = np.random.default_rng(99)
    budget = HOST_CHUNK_BYTES // n
    phase = []
    for k, ty in enumerate((types, new)):
        data = [mixed_stream(O, ty[s], s, k) if k == 0 or s in moved else None for s in range(n)]
        lens = [0 if x is None else len(x) for x in data]
        cuts = [c[:3] if k == 0 else c for c in fleet_cuts(rng, lens, budget)]
        pieces, _ = _pieces_from_cuts([np.zeros(0, np.uint8) if x is None else x for x in data], cuts)
        phase.append(pieces)
    # phase 0: three pushes of each stream's first bytes; phase 1: the moved streams' new bytes, the others' rest
    moved_set = set(moved)
    rest = [None if s in moved_set else mixed_stream(O, types[s], s, 0)[sum(len(p[s]) for p in phase[0]):]
            for s in range(n)]
    later = [[phase[1][t][s] if s in moved_set else rest[s][t * budget // 2:(t + 1) * budget // 2] for s in range(n)]
             for t in range(max(len(phase[1]), 3))]
    pieces = phase[0] + later
    stride = max(1, max(len(p) for push in pieces for p in push))
    assert stride <= budget
    rx = receive_times(rng, "bytes", None, pieces, stride)
    ctx = R.Context(0, MAX_NODES, n * MS)
    sess = R.MixedByteStreamSession(ctx, types, stride, MAX_NODES, MS)
    big = Drive.__new__(Drive)
    big.R, big.kind, big.ans, big.n, big.stride, big.max_nodes, big.ms, big.sess = \
        R, "bytes", 0, n, stride, MAX_NODES, MS, sess
    before = Blocks(R, ctx, types, range(n), stride)
    prm, cprm, timing = R.scan_params(*PARAMS), R.cloud_params(**CLOUD, is_new_protocol=PARAMS[0]), R.Timing(*TIMING)
    after = None
    for t, push in enumerate(pieces):
        if t == len(phase[0]):
            held = M.state(R, sess)
            ct0 = sess.counters().copy()
            sess.set_answer_types(new, np.array([s in moved_set for s in range(n)], np.uint8))
            assert sess.ans_types.tolist() == new
            st = M.state(R, sess)
            for s in range(n):
                assert [a[s] for a in st] == ([0, 0, 0] if s in moved_set else [a[s] for a in held]), s
            assert sess.counters().tobytes() == ct0.tobytes()
            after = Blocks(R, ctx, new, moved, stride)
        got = big.push(push, prm, "host_ts", timing, rx[t])
        exp = before.push(push, prm, "host_ts", timing, rx[t], moved_set if after else ())
        if after:
            exp.update(after.push(push, prm, "host_ts", timing, rx[t], ()))
        for s in range(n):
            assert slots(got, s, MS) == exp[s], (t, s)
    # the reads of the last push, and the counters of both sessions of a moved stream
    ct = sess.counters()
    xc = sess.cloud(cprm)
    fl = sess.laserscan_msgs(prm, 1234)
    for ref in (after, before):
        for d, part in ref.drives:
            oc, om = d.sess.counters(), d.sess.cloud(cprm)
            ol = d.sess.laserscan_msgs(prm, 1234)
            for j, s in enumerate(part):
                if ref is before and s in moved_set:
                    continue
                extra = 0 if ref is before else before.at[s][0].sess.counters()[before.at[s][1]]
                row = oc[j] if ref is before else np.array(tuple(int(a) + int(b) for a, b in zip(oc[j], extra)),
                                                            oc.dtype)
                assert ct[s].tobytes() == np.asarray(row, oc.dtype).tobytes(), ("counters", s)
                sl, ol_sl = slice(s * MS, (s + 1) * MS), slice(j * MS, (j + 1) * MS)
                assert xc["point_counts"][sl].tolist() == om["point_counts"][ol_sl].tolist(), ("cloud", s)
                for i in range(MS):
                    c = int(om["point_counts"][j * MS + i])
                    assert xc["xyzi"][s * MS + i, :c].tobytes() == om["xyzi"][j * MS + i, :c].tobytes(), ("cloud", s)
                assert fl[sl] == ol[ol_sl], ("laserscan_msgs", s)
    before.close()
    after.close()
    sess.close()
    ctx.close()


# ---- slot tables past one tile and one grid row ----------------------------------------------------------------------
TABLE_NODES, TABLE_SCANS = 2048, 32
FRAMES = ["a", "laser", "lidar_07", "x" * 30, "abc"]


def table_stream(s):
    """a 0x81 stream of revolutions of 900..1900 nodes: 3 to 6 of them in one push"""
    return normal_stream(6000 + 17 * (s % 31), 90000 + s, nodes_per_rev=900 + 13 * (s % 77), noise=50)


def table_slots(n):
    return n * TABLE_SCANS


def test_table_session_crosses_a_grid_row_and_packs_at_70k_slots():
    """the table session has more slots than one grid row of message writers and many directory tiles; pack() of
    70000 slots puts every message where the exclusive scan of the 16-rounded sizes says"""
    _, _, n = grids(132)
    assert table_slots(n) > SLAB + 1 and table_slots(700) > 16 * 1024
    rng = np.random.default_rng(70)
    sz = rng.integers(0, 70, 70000)
    sz[rng.random(70000) < 0.4] = 0
    msgs = [bytes(int(v)) if v else None for v in sz]
    offs, sizes, total = pack(msgs)
    rounded = (sz + 15) // 16 * 16
    assert (offs == np.concatenate([[0], np.cumsum(rounded)[:-1]])).all() and (sizes == sz).all()
    last = int(np.nonzero(sz)[0][-1])
    assert total == int(offs[last]) + int(sz[last]) and offs[SLAB] == rounded[:SLAB].sum()


@gpu
@pytest.mark.parametrize("ctx_streams", ["all", 700])
def test_slot_tables_past_one_tile_and_one_grid_row(R, sizes, ctx_streams):
    """one push of n streams into a session of n * 32 > 65535 slots: every slot's message offset, size and bytes of
    both kinds (host and device), exact and one-short capacities, and the grabbed nodes' directory.  With a context of
    700 streams the host calls run over several chunks and the node directory rebases per chunk."""
    import torch

    _, _, n = sizes
    ms, ns = TABLE_SCANS, table_slots(n)
    streams = [table_stream(s) for s in range(n)]
    stride = max(len(x) for x in streams)
    ctx = R.Context(0, TABLE_NODES, (n if ctx_streams == "all" else ctx_streams) * ms)
    sess = R.NormalStreamSession(ctx, n, stride, TABLE_NODES, ms)
    frames = [FRAMES[s % len(FRAMES)] for s in range(n)]
    rmax = (8.0 + (np.arange(n) % 9)).astype(np.float32)
    sess.set_frames(frames, rmax)
    buf = np.full((n, stride), 0xEE, np.uint8)
    for s, x in enumerate(streams):
        buf[s, :len(x)] = x
    prm = R.scan_params(*PARAMS)
    out = sess.push(buf, np.array([len(x) for x in streams], np.uint32), prm)
    sps = out["scans_per_stream"]
    assert (sps >= 2).all() and (sps <= ms).all()
    # LaserScan messages: the builder on the push's outputs, unstamped
    exp = []
    for i in range(ns):
        s, k = divmod(i, ms)
        m = int(out["beam_counts"][i])
        exp.append(None if k >= int(sps[s]) or m == 0 else
                   expected_laserscan(frames[s], rmax[s], 0, 0, 0, False, out["ranges"][i, :m],
                                      out["intensities"][i, :m], out["angle_increment"][i]))
    for lo in (1024, 2048, 3072, SLAB - 1, SLAB, SLAB + 1, ns - ms):
        assert any(exp[i] is not None for i in range(lo, lo + ms)), lo
    cprm = R.cloud_params(**CLOUD, is_new_protocol=PARAMS[0])
    xyzi = torch.zeros((ns, TABLE_NODES, 4), dtype=torch.float32, device="cuda")
    pcount = torch.zeros(ns, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    sess.cloud_dev(cprm, xyzi.data_ptr(), pcount.data_ptr())
    ctx.synchronize()
    pc = pcount.cpu().numpy()
    used = [i for i in range(ns) if i % ms < int(sps[i // ms])]
    top = max(1, int(pc.max()))
    rows = xyzi[torch.as_tensor(used, device="cuda"), :top].cpu().numpy()
    exp_c = [None] * ns
    for r, i in enumerate(used):
        exp_c[i] = expected_cloud(frames[i // ms], 0, 0, rows[r, :pc[i]])
    del xyzi, rows
    for kind, e, p in (("laserscan", exp, prm), ("cloud", exp_c, cprm)):
        _, _, total = pack(e)
        host = sess.laserscan_msgs if kind == "laserscan" else sess.cloud_msgs
        got = host(p, 0, msgs=np.full(total, 0x5A, np.uint8), packed=True)
        assert got["result"] == 0, kind
        check_packed(got, e)
        short = host(p, 0, msgs=np.full(total - 1, 0x5A, np.uint8), packed=True)
        assert short["result"] == R.capi.RESULT_INSUFFICIENT_MEMORY and short["total_bytes"] == total, kind
        assert (short["msg_sizes"] == 0).all() and (short["msgs"] == 0x5A).all(), kind
        check_packed(dev_msgs(R, sess, kind, p, 0, total), e, 0xA5)
        d = dev_msgs(R, sess, kind, p, 0, total - 1)
        assert d["total_bytes"] == total and (d["msg_sizes"] == 0).all() and (d["msgs"] == 0xA5).all(), kind
    # grabbed nodes: the directory's offsets, counts and statuses, exact and one-short capacities, host and device
    probe = sess.nodes(packed=True, nodes=np.zeros(2, R.NODE_DTYPE))
    total = probe["total_nodes"]
    assert probe["result"] == R.capi.RESULT_INSUFFICIENT_MEMORY and total > 0
    full = sess.nodes(packed=True, nodes=np.zeros(total, R.NODE_DTYPE))
    assert full["result"] == 0 and full["total_nodes"] == total
    check_packing(full, ns)
    counts = full["node_counts"]
    k_of = np.arange(ns) % ms
    live = k_of < np.repeat(sps, ms)
    assert (counts[~live] == 0).all() and (counts[live] > 0).all()
    assert counts[SLAB:].sum() > 0 and (counts[:1024] > 0).any()
    dn = dev_nodes(torch, sess, capacity=total)
    for k in ("node_offsets", "node_counts", "status"):
        assert (dn[k] == full[k]).all(), k
    assert dn["total_nodes"] == total
    host = full["nodes"].view(np.uint64)
    for i in np.nonzero(counts)[0].tolist():
        o, c = int(full["node_offsets"][i]), int(counts[i])
        assert dn["nodes"][o:o + c].tobytes() == host[o:o + c].tobytes(), ("nodes_dev", i)
    assert (dn["nodes"][total:] == np.uint64(2**64 - 7)).all()
    short = dev_nodes(torch, sess, capacity=total - 1)
    assert short["total_nodes"] == total and (short["node_counts"] == 0).all()
    sess.close()
    ctx.close()


# ---- stateless launches past 65535 grid rows -------------------------------------------------------------------------
def named(bad):
    """the first wrong streams, the boundary ones by name"""
    return {"first": bad[:8], "around 65535": [s for s in bad if SLAB - 2 <= s <= SLAB + 2], "n": len(bad)}


@gpu
def test_node_timestamps_every_stream_past_65535(R, oracle):
    import torch

    O, ans, per, stride = oracle, 0x84, 96, 2
    n = SLAB + 2 + 300
    rng = np.random.default_rng(81)
    caps = format_stream(O, ans, n * stride, 5, sync_every=37).reshape(n, stride, CB[ans])
    counts = rng.integers(1, stride + 1, n).astype(np.uint32)
    counts[[SLAB - 1, SLAB, SLAB + 1, n - 1]] = stride
    rx = rx_times(n * stride, 12).reshape(n, stride)
    timing = (63, 256000, 17, 0)
    dec = [O.decode_capsules(ans, caps[s, :counts[s]], timing[0]) for s in range(n)]
    status = np.zeros((n, stride), np.uint32)
    offs = np.zeros((n, stride), np.uint32)
    for s, (_, st, of, _) in enumerate(dec):
        status[s, :counts[s]] = st
        offs[s, :counts[s]] = of
    d = {k: torch.from_numpy(np.ascontiguousarray(v).view(np.int32 if v.dtype == np.uint32 else np.int64)).cuda()
         for k, v in (("status", status), ("offs", offs), ("counts", counts), ("rx", rx.astype(np.uint64)))}
    ts = torch.full((n, stride * per), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    with R.Context(0, 4096, 1) as ctx:
        ctx.node_timestamps_dev(ans, R.Timing(*timing), d["rx"].data_ptr(), d["status"].data_ptr(),
                                d["offs"].data_ptr(), d["counts"].data_ptr(), n, stride, ts.data_ptr())
        ctx.synchronize()
    got = ts.cpu().numpy().view(np.uint64)
    t4 = O.timing4(*timing)
    bad = []
    for s in range(n):
        nodes, st, of, _ = dec[s]
        e = O.node_timestamps(ans, t4, rx[s, :counts[s]], st, of, len(nodes))
        if not ((got[s, :len(nodes)] == e).all() and (got[s, len(nodes):] == np.uint64(2**64 - 1)).all()):
            bad.append(s)
    assert not bad, named(bad)
    assert sum(len(x[0]) > 0 for x in dec[SLAB:]) > 100


@gpu
def test_normal_timestamps_every_stream_past_65535(R, oracle):
    import torch

    O = oracle
    n = SLAB + 2 + 300
    rng = np.random.default_rng(82)
    stride, chunk = 25, 8
    stride_chunks = -(-stride // chunk)
    recs = standard_records(rng, n * 5).reshape(n, stride)
    counts = np.array([5 * int(rng.integers(1, 6)) - (int(rng.integers(0, 3)) if s % 3 == 0 else 0) for s in range(n)],
                      np.uint32)
    counts[[SLAB - 1, SLAB, SLAB + 1, n - 1]] = stride
    rx = rx_times(n * stride_chunks, 13).reshape(n, stride_chunks)
    timing = (476, 115200, 250, 0)
    dec = [O.decode_normal(recs[s, :counts[s]]) for s in range(n)]
    ends = np.zeros((n, stride // 5), np.uint32)
    ncount = np.zeros(n, np.uint32)
    for s, (nodes, e, _) in enumerate(dec):
        ends[s, :len(nodes)] = e
        ncount[s] = len(nodes)
    ts = torch.full((n, stride // 5), -1, dtype=torch.int64, device="cuda")
    d_ends = torch.from_numpy(ends.view(np.int32)).cuda()
    d_cnt = torch.from_numpy(ncount.view(np.int32)).cuda()
    d_rx = torch.from_numpy(rx.astype(np.uint64).view(np.int64)).cuda()
    torch.cuda.synchronize()
    with R.Context(0, 4096, 1) as ctx:
        ctx.normal_timestamps_dev(R.Timing(*timing), d_ends.data_ptr(), d_cnt.data_ptr(), n, stride // 5, chunk,
                                  d_rx.data_ptr(), stride_chunks, ts.data_ptr())
        ctx.synchronize()
    got = ts.cpu().numpy().view(np.uint64)
    t4 = O.timing4(*timing)
    bad = []
    for s in range(n):
        m = int(ncount[s])
        e = O.normal_timestamps(t4, dec[s][1], chunk, rx[s])
        if not ((got[s, :m] == e).all() and (got[s, m:] == np.uint64(2**64 - 1)).all()):
            bad.append(s)
    assert not bad, named(bad)
    assert ncount[SLAB:].sum() > 100


@gpu
def test_laserscan_cdr_every_scan_past_65535(R):
    import torch

    n, stride, frame_id = SLAB + 2 + 500, 6, "laser_frame_9"
    rng = np.random.default_rng(83)
    ranges = (rng.random((n, stride)) * 40).astype(np.float32)
    intens = rng.integers(0, 256, (n, stride)).astype(np.float32)
    beams = rng.integers(0, stride + 1, n).astype(np.uint32)
    beams[[SLAB - 1, SLAB, SLAB + 1, n - 1]] = stride
    inc = rng.random(n).astype(np.float32)
    meta = np.zeros(n, R.capi.LASERSCAN_META_DTYPE)
    meta["stamp_sec"] = rng.integers(-5, 2_000_000_000, n)
    meta["stamp_nanosec"] = rng.integers(0, 1_000_000_000, n)
    for k in ("angle_min", "angle_max", "angle_increment", "time_increment", "scan_time", "range_min", "range_max"):
        meta[k] = rng.random(n).astype(np.float32)
    cdr_stride = (R.lib().rpl_laserscan_cdr_size(len(frame_id), stride) + 15) & ~15
    out = torch.full((n, cdr_stride), 0xEE, dtype=torch.uint8, device="cuda")
    sz = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d = [torch.from_numpy(a).cuda() for a in (ranges, intens, beams.view(np.int32), inc, meta.view(np.uint8))]
    torch.cuda.synchronize()
    with R.Context(0, 4096, 1) as ctx:
        ctx.laserscan_cdr_batch_dev(d[4].data_ptr(), frame_id, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), n,
                                    stride, out.data_ptr(), cdr_stride, cdr_sizes=sz.data_ptr(),
                                    angle_increment=d[3].data_ptr())
        ctx.synchronize()
    ho, hs = out.cpu().numpy(), sz.cpu().numpy()
    bad = []
    for s in range(n):
        m, b = meta[s], int(beams[s])
        e = cdr.laserscan_cdr(int(m["stamp_sec"]), int(m["stamp_nanosec"]), frame_id,
                              [m["angle_min"], m["angle_max"], inc[s], m["time_increment"], m["scan_time"],
                               m["range_min"], m["range_max"]], ranges[s, :b], intens[s, :b])
        if not (hs[s] == len(e) and ho[s, :len(e)].tobytes() == e and (ho[s, len(e):] == 0xEE).all()):
            bad.append(s)
    assert not bad, named(bad)


@gpu
def test_pointcloud2_cdr_every_cloud_past_65535(R):
    import torch

    n, stride, frame_id = SLAB + 2 + 500, 3, "lidar_3"
    rng = np.random.default_rng(84)
    xyzi = rng.normal(0, 10, (n, stride, 4)).astype(np.float32)
    pcount = rng.integers(0, stride + 1, n).astype(np.uint32)
    pcount[[SLAB - 1, SLAB, SLAB + 1, n - 1]] = stride
    stamps = np.stack([rng.integers(0, 2**31, n), rng.integers(0, 10**9, n)], axis=1).astype(np.uint32)
    cdr_stride = (R.lib().rpl_pointcloud2_cdr_size(len(frame_id), stride) + 15) & ~15
    out = torch.full((n, cdr_stride), 0xEE, dtype=torch.uint8, device="cuda")
    sz = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d = [torch.from_numpy(a).cuda() for a in (xyzi, pcount.view(np.int32), stamps.view(np.int32))]
    torch.cuda.synchronize()
    with R.Context(0, 4096, 1) as ctx:
        ctx.pointcloud2_cdr_batch_dev(d[2].data_ptr(), frame_id, d[0].data_ptr(), d[1].data_ptr(), n, stride,
                                      out.data_ptr(), cdr_stride, cdr_sizes=sz.data_ptr())
        ctx.synchronize()
    ho, hs = out.cpu().numpy(), sz.cpu().numpy()
    bad = []
    for s in range(n):
        e = cdr.pointcloud2_cdr(int(stamps[s, 0]), int(stamps[s, 1]), frame_id, xyzi[s, :pcount[s]])
        if not (hs[s] == len(e) and ho[s, :len(e)].tobytes() == e and (ho[s, len(e):] == 0xEE).all()):
            bad.append(s)
    assert not bad, named(bad)


# ---- the grids, from the profiler's trace ----------------------------------------------------------------------------
PROFILED = [("bytes", 0x82), ("bytes", 0x83), ("normal", 0x81), ("framed", 0x85), ("framed", 0x86)]


def profiled_grids():
    """{kind: [(kernel, CTAs, streams)]}: one push and one host nodes call of a fleet of every PROFILED kind, under
    the CUDA profiler; each launch's grid from the exported trace (run in a child process)"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    import rplidar_ros2_driver_b200 as R
    from oracle import pyoracle as O

    _, _, n = grids(torch.cuda.get_device_properties(0).multi_processor_count)
    res = {}
    for kind, ans in PROFILED:
        streams, pieces, stride = fleet_pieces(O, kind, ans, n, 5)
        with R.Context(0, MAX_NODES, n * MS) as ctx:
            d = Drive(R, ctx, kind, ans, n, stride, MAX_NODES, MS)
            d.push(pieces[0], R.scan_params(*PARAMS), "host")
            with tempfile.TemporaryDirectory() as tmp:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    d.push(pieces[1], R.scan_params(*PARAMS), "dev")
                    d.sess.nodes(apply_ascend=False)
                    torch.cuda.synchronize()
                    torch.cuda._sleep(50_000_000)  # keep the last launch clear of the capture window's edge
                    torch.cuda.synchronize()
                path = os.path.join(tmp, "trace.json")
                prof.export_chrome_trace(path)
                with open(path) as f:
                    events = json.load(f)["traceEvents"]
            d.close()
        res[f"{kind}_{ans:02x}"] = [(e["name"], int(np.prod(e["args"]["grid"])), n) for e in events
                                    if e.get("cat") == "kernel" and "grid" in e.get("args", {})]
    return res


@gpu
def test_launches_have_fewer_ctas_than_streams():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"),
                                                       os.environ.get("PYTHONPATH", "")]))
    code = "import json, test_gpu_fleet_scale as T; print('GRIDS ' + json.dumps(T.profiled_grids()), flush=True)"
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, env=env, capture_output=True, text=True,
                       timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("GRIDS ")]
    assert r.returncode == 0 and lines, f"the profiling process failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    got = json.loads(lines[-1][len("GRIDS "):])
    print(json.dumps({k: sorted({(name.split("(")[0][:60], g) for name, g, _ in v}) for k, v in got.items()}))
    for kind, launches in got.items():
        want = ["decode_", "assemble_"] + (["frame_capsules_kernel"] if kind.startswith("bytes") else [])
        for w in want:
            hit = [(name, g, n) for name, g, n in launches if w in name]
            assert hit, (kind, w, sorted({x[0][:60] for x in launches}))
            assert all(g < n for _, g, n in hit), (kind, hit)
    # the gather runs only when the profiled push published scans (an HQ push of under one revolution publishes none)
    gather = [(kind, g, n) for kind, v in got.items() for name, g, n in v if "node_gather_kernel" in name]
    assert gather and all(g < n for _, g, n in gather), gather
