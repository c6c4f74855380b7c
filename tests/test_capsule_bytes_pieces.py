"""The contract of the capsule byte sessions (rpl_capsule_stream_create_bytes), pinned on the CPU for express (0x82),
HQ (0x83), ultra (0x84), dense (0x85) and ultra-dense (0x86): the SDK's own unpacker fed a DAMAGED raw byte stream in
pieces (its search for the sync bytes carried from one piece to the next), then its own ScanDataHolder, publishes
exactly the scans -- and, with its clock set per piece, the scan-begin stamps -- that the restatement publishes from
the whole stream in one call: framing (frame_stream below) -> oracle capsule decoder -> holder restatement, each frame
stamped with the receive time of its last byte.  The sessions (tests/test_gpu_capsule_byte_stream.py) are held to the
restatement, so "any split of the bytes into pushes gives the whole stream's scans" is the SDK's behaviour and not a new
definition.  frame_stream restates the framing with the HQ rule (handler_hqnode.cpp:95-172: a byte other than 0xA5 is
skipped while waiting, and changes nothing), which the oracle framer does not serve; for the other formats it is held
to the oracle framer here.  Needs the compiled reference (oracle/_ref); skipped without it.

The stream builders here are shared with the GPU test."""
import numpy as np
import pytest

from test_capsule_stream_pieces import format_stream
from test_timestamps_vs_ref import TIMINGS

FORMATS = [0x82, 0x83, 0x84, 0x85, 0x86]
MAX_NODES, MAX_SCANS = 2048, 64


def frame_stream(O, ans, b):
    """The unpackers' search for the sync bytes as a function of the whole stream: (capsules [m, frame size], last
    [m] index of each capsule's last byte, bytes left in an unfinished frame).  Every run of skipped bytes in front of a
    frame becomes one all-zero capsule (its `last` is the frame's); HQ skips without a trace."""
    cb = O.capsule_bytes(ans)
    b = np.asarray(b, np.uint8)
    n, q, lost = len(b), 0, False
    caps, last = [], []
    while q < n:
        if ans == 0x83:
            if b[q] != 0xA5:
                q += 1
                continue
        else:
            if (b[q] >> 4) != 0xA:
                lost, q = True, q + 1
                continue
            if q + 1 >= n:
                break
            if (b[q + 1] >> 4) != 0x5:
                lost, q = True, q + 2
                continue
        if q + cb > n:
            break
        if lost:
            caps.append(np.zeros(cb, np.uint8))
            last.append(q + cb - 1)
            lost = False
        caps.append(b[q:q + cb])
        last.append(q + cb - 1)
        q += cb
    out = np.stack(caps) if caps else np.zeros((0, cb), np.uint8)
    return out, np.array(last, np.int64), n - min(q, n)


def raw_stream(O, ans, seed, n_caps=None, edits=12):
    """one damaged raw byte stream: dropped, inserted and flipped bytes, false first markers (HQ: 0xA5) and false
    marker pairs inside skipped runs, noise runs, and at random a truncated tail"""
    rng = np.random.default_rng(seed)
    n_caps = n_caps or (150 if ans == 0x83 else 500)
    caps = format_stream(O, ans, n_caps, seed, sync_every=120 + seed % 50, bad=False)
    cb = caps.shape[1]
    raw = bytearray(caps.reshape(-1).tobytes())
    first = 0xA5 if ans == 0x83 else 0xA0
    for _ in range(edits):
        p = int(rng.integers(0, len(raw)))
        kind = int(rng.integers(0, 6))
        if kind == 0:
            del raw[p: p + int(rng.integers(1, 5))]
        elif kind == 1:
            raw[p:p] = bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8))
        elif kind == 2:
            raw[p] ^= int(rng.integers(1, 256))
        elif kind == 3:  # a skipped run with false first markers and marker pairs in it
            run = rng.integers(0, 0xA0, int(rng.integers(3, 40)), dtype=np.uint8)
            run[rng.random(len(run)) < 0.3] = first | (0 if ans == 0x83 else int(rng.integers(0, 16)))
            raw[p:p] = bytes(run)
            raw[p:p] = bytes([0xA0 | int(rng.integers(0, 16)), 0x50 | int(rng.integers(0, 16))])
        elif kind == 4:  # noise
            raw[p:p] = bytes(rng.integers(0, 256, int(rng.integers(50, 3 * cb)), dtype=np.uint8))
        else:  # a lone first marker right where a frame starts
            raw[p - p % cb: p - p % cb] = bytes([first | (0 if ans == 0x83 else 3)])
    if rng.random() < 0.5:
        del raw[len(raw) - int(rng.integers(1, cb)):]
    return np.frombuffer(bytes(raw), np.uint8).copy()


def restated(O, ans, b, sample_duration_us=31):
    """(nodes, status, offsets, last byte of each capsule): framing -> oracle decoder on the whole stream"""
    caps, last, _ = frame_stream(O, ans, b)
    nodes, status, offs, _ = O.decode_capsules(ans, caps, sample_duration_us)
    return nodes, status, offs, last


def restated_scans(O, ans, b, max_nodes=MAX_NODES, max_scans=MAX_SCANS):
    nodes, status, offs, _ = restated(O, ans, b)
    return O.assemble_scans(nodes, O.resets_from_capsules(status, offs), max_nodes, max_scans)


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_ref() and oracle.have_ref_holder() and oracle.have_ref_clock()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle


def _pieces(cb, piece):
    return {"1": 1, "2": 2, "cb-1": cb - 1, "cb": cb, "cb+1": cb + 1, "3cb+7": 3 * cb + 7, "whole": 0}[piece]


@pytest.mark.parametrize("ans", [0x82, 0x84, 0x85, 0x86])
def test_frame_stream_is_the_oracle_framer(oracle, ans):
    for seed in range(6):
        b = raw_stream(oracle, ans, 300 + seed)
        caps, last, left = frame_stream(oracle, ans, b)
        exp, eleft = oracle.frame_capsules(ans, b)
        assert caps.shape == exp.shape and (caps == exp).all() and left == eleft, (hex(ans), seed)
        assert (np.diff(last) >= 0).all()


@pytest.mark.parametrize("ans", FORMATS)
@pytest.mark.parametrize("piece", ["1", "2", "cb-1", "cb", "cb+1", "3cb+7", "whole"])
def test_sdk_fed_bytes_in_pieces_publishes_the_restated_scans(O, ans, piece):
    cb = O.capsule_bytes(ans)
    chunk = _pieces(cb, piece)
    damaged = published = 0
    for seed in (41, 42, 43):
        b = raw_stream(O, ans, seed + ans)
        rn, ev = O.ref_unpack(ans, b, 31, chunk)
        rs, rl, rk = O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), MAX_NODES, MAX_SCANS)
        nodes, status, offs, _ = restated(O, ans, b)
        assert len(rn) == len(nodes) and (rn.view(np.uint64) == nodes.view(np.uint64)).all(), (hex(ans), seed)
        es, el, ek = O.assemble_scans(nodes, O.resets_from_capsules(status, offs), MAX_NODES, MAX_SCANS)
        assert rk == ek and (rl == el).all(), (hex(ans), seed, rk, ek)
        published += ek
        for k in range(min(ek, MAX_SCANS)):
            assert (rs[k, : rl[k]].view(np.uint64) == es[k, : el[k]].view(np.uint64)).all(), (hex(ans), chunk, k)
        damaged += int(((status & (O.CAPSULE_BAD_FRAME | O.CAPSULE_CHECKSUM_ERR)) != 0).any())
    assert damaged >= 2 and published >= 3


@pytest.mark.parametrize("ans", FORMATS)
@pytest.mark.parametrize("piece", ["1", "2", "cb-1", "cb", "cb+1", "3cb+7", "whole"])
def test_sdk_fed_bytes_in_pieces_stamps_the_restated_scans(O, ans, piece):
    cb = O.capsule_bytes(ans)
    published = 0
    for i, seed in enumerate((51, 52)):
        b = raw_stream(O, ans, seed + ans)
        chunk = _pieces(cb, piece) or len(b)
        timing = TIMINGS[(i + ans) % len(TIMINGS)]
        if ans != 0x83:
            timing = (31,) + tuple(timing[1:])  # the streams' revolutions are built for the 31 us jump threshold
        t4 = O.timing4(*timing)
        n_pieces = -(-len(b) // chunk)
        rng = np.random.default_rng(seed)
        rx = (10_000_000 + np.cumsum(rng.integers(1, 3000, n_pieces))).astype(np.uint64)
        rnodes, rts = O.ref_unpack_ts(ans, b, chunk, rx, t4)
        _, ev = O.ref_unpack(ans, b, int(t4[0]), chunk)
        _, rl, rk, rsts = O.ref_assemble_scans_ts(rnodes, rts, ev[ev[:, 0] == 1, 1].astype(np.uint32), MAX_NODES,
                                                  MAX_SCANS)
        nodes, status, offs, last = restated(O, ans, b, int(t4[0]))
        ts = O.node_timestamps(ans, t4, rx[last // chunk], status, offs, len(nodes))
        _, el, ek, ests = O.assemble_scans_ts(nodes, ts, O.resets_from_capsules(status, offs), MAX_NODES, MAX_SCANS)
        assert rk == ek and (rl[:rk] == el[:ek]).all(), (rk, ek)
        published += ek
        assert (rsts[:rk] == ests[:ek]).all(), (hex(ans), chunk, np.flatnonzero(rsts[:rk] != ests[:ek])[:5])
    assert published >= 2
