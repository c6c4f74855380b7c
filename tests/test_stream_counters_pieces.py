"""The stream sessions' counters (rpl_capsule_stream_counters), restated on a whole stream and pinned against the SDK on
the CPU.  The restatement: the framing restated by frame_stream (held to the oracle framer frame for frame by
tests/test_capsule_bytes_pieces.py) or the oracle's 0x81 byte machine, then the oracle decoder's capsule statuses, then
a ScanDataHolder restatement that also counts what it drops.  Pinned as follows:
  * the event counts (checksum errors, encoder resets, scan resets, nodes) are those of the SDK's own unpacker fed the
    damaged raw streams of all six answer types in pieces of 1, 2, frame - 1, frame, frame + 1 and 3 * frame + 7 bytes;
  * the holder restatement publishes the scans of the SDK's own ScanDataHolder, and its counters are checked against
    hand-built cases, one per rule (sl_lidar_driver.cpp:272-315).
Without the compiled reference (oracle/_ref) the SDK's outputs recorded in tests/golden/stream_counters_golden.npz
(tests/golden/make_stream_counters_golden.py) stand in for it.  tests/test_gpu_stream_counters.py holds the sessions to
the restatement."""
import hashlib
import os

import numpy as np
import pytest

from test_capsule_bytes_pieces import frame_stream, raw_stream
from test_normal_stream_pieces import normal_stream

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_counters_golden.npz")
ALL_TYPES = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
PIECES = ["1", "2", "cb-1", "cb", "cb+1", "3cb+7"]
FIELDS = ("bytes_in", "frames", "skipped_bytes", "bad_frames", "checksum_errors", "encoder_resets", "scan_resets",
          "discarded_capsules", "nodes", "nodes_unopened", "nodes_overwritten", "scans_rewound", "scans_published",
          "scans_unreturned")
ERR_ENCODER_RESET, ERR_CHECKSUM = 0x8001, 0x8002  # dataunpacker.h:63-64


def frame_size(O, ans):
    return 5 if ans == 0x81 else O.capsule_bytes(ans)


def golden_stream(O, ans, seed):
    """a damaged raw stream of the answer type (0x81: records with failed checks, dropped, inserted and noise bytes)"""
    return normal_stream(6000, seed) if ans == 0x81 else raw_stream(O, ans, seed)


def stream_digest(b):
    return hashlib.sha256(np.ascontiguousarray(b, np.uint8).tobytes()).digest()


def holder(nodes, resets, max_nodes):
    """ScanDataHolder::pushScanNodeData / rewindCurrentScanData (sl_lidar_driver.cpp:272-315) node by node, counting:
    (published scan lengths, {nodes_unopened, nodes_overwritten, scans_rewound, scans_published}).  resets: node
    positions of the scan-reset requests, each made before the node at its position (at len(nodes): after the last)."""
    sync = (np.asarray(nodes).view(np.uint64) >> np.uint64(56)) & np.uint64(1)
    resets = np.sort(np.asarray(resets, np.int64))
    size, ri, lens = 0, 0, []
    c = dict(nodes_unopened=0, nodes_overwritten=0, scans_rewound=0, scans_published=0)

    def rewind_upto(x):
        nonlocal size, ri
        while ri < len(resets) and resets[ri] <= x:
            if size:
                c["scans_rewound"] += 1
            size, ri = 0, ri + 1

    for i, f in enumerate(sync.tolist()):
        rewind_upto(i)
        if f:
            if size:
                lens.append(min(size, max_nodes))
                c["scans_published"] += 1
            size = 0
        elif size == 0:
            c["nodes_unopened"] += 1
            continue
        if size >= max_nodes:
            c["nodes_overwritten"] += 1
        else:
            size += 1
    rewind_upto(len(sync))
    return lens, c


def status_counts(O, status):
    return dict(bad_frames=int(((status & O.CAPSULE_BAD_FRAME) != 0).sum()),
                checksum_errors=int(((status & O.CAPSULE_CHECKSUM_ERR) != 0).sum()),
                encoder_resets=int(((status & O.CAPSULE_ENCODER_RESET_ERR) != 0).sum()),
                scan_resets=int(((status & O.CAPSULE_SYNC) != 0).sum()),
                discarded_capsules=int(((status & O.CAPSULE_DISCARD) != 0).sum()))


def restated_counters(O, ans, data, max_nodes, byte_session=True, sample_duration_us=31):
    """The counters a session of answer type ans (max_nodes) reaches on the whole stream `data` (a byte session's raw
    bytes, or a framed session's capsules [m, frame size]), scans_unreturned aside (it depends on the pushes); also
    the published scan lengths.  held_bytes: what the session holds at the end."""
    c = dict.fromkeys(FIELDS, 0)
    if ans == 0x81:
        nodes, _, held = O.decode_normal(data)
        c.update(bytes_in=len(data), frames=len(nodes), skipped_bytes=len(data) - 5 * len(nodes) - held)
        resets = np.zeros(0, np.int64)
    else:
        cb = O.capsule_bytes(ans)
        if byte_session:
            caps, _, held = frame_stream(O, ans, data)
            frames = int((caps != 0).any(axis=1).sum())  # a frame starts with its sync byte: never all zero
            c.update(bytes_in=len(data), frames=frames, skipped_bytes=len(data) - cb * frames - held)
        else:
            caps, held = np.asarray(data, np.uint8).reshape(-1, cb), 0
            c.update(bytes_in=caps.size, frames=len(caps))
        nodes, status, offs, _ = O.decode_capsules(ans, caps, sample_duration_us)
        c.update(status_counts(O, status))
        resets = O.resets_from_capsules(status, offs)
    lens, h = holder(nodes, resets, max_nodes)
    c.update(h, nodes=len(nodes))
    return c, lens, held


def sdk_events(O, ans, b, chunk):
    """(nodes, checksum errors, encoder resets, scan resets) of the SDK's unpacker fed b `chunk` bytes at a time"""
    nodes, ev = O.ref_unpack(ans, b, 31, chunk)
    err = ev[ev[:, 0] == 2, 2]
    return (len(nodes), int((err == ERR_CHECKSUM).sum()), int((err == ERR_ENCODER_RESET).sum()),
            int((ev[:, 0] == 1).sum())), nodes, ev


def _chunk(cb, piece):
    return {"1": 1, "2": 2, "cb-1": cb - 1, "cb": cb, "cb+1": cb + 1, "3cb+7": 3 * cb + 7}[piece]


GOLDEN_SEEDS = (71, 72)
GOLDEN_MAX_NODES = 1024


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _have_ref(O):
    return O.have_ref() and O.have_ref_holder()


@pytest.mark.parametrize("ans", ALL_TYPES)
@pytest.mark.parametrize("piece", PIECES)
def test_event_counts_are_the_sdk_unpackers(oracle, golden, ans, piece):
    """checksum errors, encoder resets, scan resets and nodes of the restatement (whole stream, one pass) are the
    events the SDK's unpacker raises fed the same bytes in pieces"""
    O = oracle
    chunk = _chunk(frame_size(O, ans), piece)
    seen = np.zeros(4, np.int64)
    for seed in GOLDEN_SEEDS:
        b = golden_stream(O, ans, seed)
        key = f"{ans:02x}_{seed}"
        assert golden[f"{key}_sha256"].tobytes() == stream_digest(b), "the stream builders changed: regenerate the fixture"
        c, _, _ = restated_counters(O, ans, b, GOLDEN_MAX_NODES)
        got = (c["nodes"], c["checksum_errors"], c["encoder_resets"], c["scan_resets"])
        if _have_ref(O):
            exp, _, _ = sdk_events(O, ans, b, chunk)
            assert tuple(exp) == tuple(golden[f"{key}_events"].tolist()), (hex(ans), seed, chunk)
        else:
            exp = tuple(golden[f"{key}_events"].tolist())
        assert got == tuple(exp), (hex(ans), seed, chunk, got, exp)
        seen += np.array(got) > 0
    # the streams exercise what they count: nodes and checksum errors everywhere, scan resets and encoder resets
    # wherever the format requests them (not HQ, whose scan starts are node flags, nor 0x81)
    assert seen[0] and (ans == 0x81 or seen[1])
    assert ans in (0x81, 0x83) or (seen[2] and seen[3])


@pytest.mark.parametrize("ans", ALL_TYPES)
def test_holder_restatement_publishes_the_sdk_holders_scans(oracle, golden, ans):
    """the counting holder publishes what ScanDataHolder publishes (the SDK's nodes and reset requests fed to it)"""
    O = oracle
    for seed in GOLDEN_SEEDS:
        b = golden_stream(O, ans, seed)
        key = f"{ans:02x}_{seed}"
        c, lens, _ = restated_counters(O, ans, b, GOLDEN_MAX_NODES)
        if _have_ref(O):
            _, rn, ev = sdk_events(O, ans, b, 7)
            _, rl, rk = O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), GOLDEN_MAX_NODES, 4096)
            assert rk <= 4096
            assert (rl[:rk] == golden[f"{key}_lens"]).all(), (hex(ans), seed)
        exp = golden[f"{key}_lens"]
        assert c["scans_published"] == len(exp) and (np.array(lens, np.uint32) == exp).all(), (hex(ans), seed)
        assert c["nodes_overwritten"] > 0 and c["scans_published"] > 0, (hex(ans), seed)


def test_byte_identity_and_framed_restatement(oracle):
    """bytes_in = frames * frame size + skipped_bytes + held bytes; a framed session of the byte session's capsules
    counts the same events, no skipped bytes and no held bytes"""
    O = oracle
    for ans in ALL_TYPES:
        b = golden_stream(O, ans, 73)
        c, lens, held = restated_counters(O, ans, b, GOLDEN_MAX_NODES)
        assert c["bytes_in"] == c["frames"] * frame_size(O, ans) + c["skipped_bytes"] + held
        assert c["skipped_bytes"] > 0, hex(ans)
        if ans == 0x81:
            continue
        caps, _, _ = frame_stream(O, ans, b)
        f, flens, _ = restated_counters(O, ans, caps, GOLDEN_MAX_NODES, byte_session=False)
        assert f["frames"] == len(caps) and f["skipped_bytes"] == 0 and f["bytes_in"] == caps.size
        for k in FIELDS[3:]:
            assert f[k] == c[k], (hex(ans), k)
        assert flens == lens
        assert ans == 0x83 or c["bad_frames"] > 0


def _nodes(flags):
    """nodes with the given scan-start flags (other fields arbitrary but fixed)"""
    n = np.zeros(len(flags), np.uint64)
    n |= np.asarray(flags, np.uint64) << np.uint64(56)
    n |= (np.arange(len(flags), dtype=np.uint64) % 7) << np.uint64(16)
    return n


@pytest.mark.parametrize("case", ["before_first_start", "reset_inside", "two_resets", "exactly_max", "max_plus_1",
                                  "three_max"])
def test_holder_counters_by_rule(oracle, case):
    """one hand-built case per holder rule; the published lengths also match the oracle holder (and the SDK's)"""
    M = 8
    if case == "before_first_start":  # 5 nodes, then a revolution of 4, then the next start
        flags, resets = [0] * 5 + [1, 0, 0, 0, 1, 0], []
        exp = dict(nodes_unopened=5, nodes_overwritten=0, scans_rewound=0, scans_published=1)
    elif case == "reset_inside":  # a reset before node 8 empties the revolution opened at 5; 8, 9 find none open
        flags, resets = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], [8]
        exp = dict(nodes_unopened=2, nodes_overwritten=0, scans_rewound=1, scans_published=1)
    elif case == "two_resets":  # two resets in a row: the second finds the revolution empty
        flags, resets = [1, 0, 0, 1, 0, 0, 0, 1], [5, 5]
        exp = dict(nodes_unopened=2, nodes_overwritten=0, scans_rewound=1, scans_published=1)
    elif case == "exactly_max":
        flags, resets = [1] + [0] * (M - 1) + [1], []
        exp = dict(nodes_unopened=0, nodes_overwritten=0, scans_rewound=0, scans_published=1)
    elif case == "max_plus_1":
        flags, resets = [1] + [0] * M + [1], []
        exp = dict(nodes_unopened=0, nodes_overwritten=1, scans_rewound=0, scans_published=1)
    else:  # three_max, and a reset after the last node empties the open revolution
        flags, resets = [1] + [0] * (3 * M - 1) + [1, 0], [3 * M + 2]
        exp = dict(nodes_unopened=0, nodes_overwritten=2 * M, scans_rewound=1, scans_published=1)
    nodes = _nodes(flags).view(oracle.NODE_DTYPE)
    lens, c = holder(nodes, resets, M)
    assert c == exp, (case, c)
    _, el, ek = oracle.assemble_scans(nodes, np.array(resets, np.uint32), M, 16)
    assert ek == len(lens) and (el[:ek] == lens).all()
    if oracle.have_ref_holder():
        _, rl, rk = oracle.ref_assemble_scans(nodes, np.array(resets, np.uint32), M, 16)
        assert rk == ek and (rl[:rk] == el[:ek]).all()
