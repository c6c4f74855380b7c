"""The contract of the stream sessions' stamped pushes, pinned on the CPU for all six answer types: the SDK's own
unpacker fed a stream in byte pieces with its clock set per piece, then its own ScanDataHolder, stamps every published
scan exactly as the restatement does on the whole stream in one call -- decoder -> per-node stamps
(oracle/timestamp_oracle.cpp) -> holder with stamps, each capsule with the receive time of the piece that delivered its
last byte (0x81: each byte with its piece's).  The sessions (tests/test_gpu_stream_stamps.py) are held to the latter,
so "the stamps of any split into pushes are the whole stream's" is the SDK's behaviour and not a new definition.  Needs
the compiled reference (oracle/_ref); skipped without it."""
import numpy as np
import pytest

from test_capsule_stream_pieces import format_stream
from test_decode_oracle_vs_ref import make_stream
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS

FORMATS = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
MAX_NODES, MAX_SCANS = 2048, 64


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_ref() and oracle.have_ref_holder() and oracle.have_ref_clock()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle


def _stream(O, ans, seed):
    """raw bytes of one stream with checksum errors and (but HQ, 0x81) scan-start capsules"""
    if ans == 0x81:
        return normal_stream(9000, seed, nodes_per_rev=1500, noise=40)
    if ans == 0x85:
        caps = make_stream(O, 600, 80.0, seed=seed, sync_every=250)
        rng = np.random.default_rng(seed)
        caps[rng.choice(600, 10, replace=False), 10] ^= 0x40
        caps[rng.choice(600, 5, replace=False)] = 0
    else:
        caps = format_stream(O, ans, 200 if ans == 0x83 else 600, seed, sync_every=250)
    return caps.reshape(-1)


def _restated(O, ans, b, t4, rx_byte):
    """the restatement's scan-begin stamps of the whole stream, every byte with its receive time"""
    if ans == 0x81:
        nodes, ends, _ = O.decode_normal(b)
        ts = O.normal_timestamps(t4, ends, 1, rx_byte)
        resets = None
    else:
        cb = O.capsule_bytes(ans)
        caps = b.reshape(-1, cb)
        nodes, status, offs, _ = O.decode_capsules(ans, caps, int(t4[0]))
        ts = O.node_timestamps(ans, t4, rx_byte[cb - 1::cb], status, offs, len(nodes))  # the capsule's last byte
        resets = O.resets_from_capsules(status, offs)
    _, lens, k, sts = O.assemble_scans_ts(nodes, ts, resets, MAX_NODES, MAX_SCANS)
    return lens[:k], sts[:k]


@pytest.mark.parametrize("ans", FORMATS)
@pytest.mark.parametrize("piece", ["1", "7", "cb-1", "cb+1", "3cb+7", "whole"])
def test_sdk_fed_in_pieces_stamps_the_whole_streams_scans(O, ans, piece):
    cb = 5 if ans == 0x81 else O.capsule_bytes(ans)
    for i, seed in enumerate((61, 62)):
        b = _stream(O, ans, seed + ans)
        chunk = {"1": 1, "7": 7, "cb-1": cb - 1, "cb+1": cb + 1, "3cb+7": 3 * cb + 7, "whole": len(b)}[piece]
        timing = TIMINGS[(i + ans) % len(TIMINGS)] if i == 0 else TIMINGS[4]  # the Ethernet interface included
        if ans != 0x83:
            timing = (31,) + tuple(timing[1:])  # the streams' revolutions are built for the 31 us jump threshold
        t4 = O.timing4(*timing)
        n_pieces = -(-len(b) // chunk)
        rng = np.random.default_rng(seed)
        rx = (10_000_000 + np.cumsum(rng.integers(1, 3000, n_pieces))).astype(np.uint64)
        rnodes, rts = O.ref_unpack_ts(ans, b, chunk, rx, t4)
        _, ev = O.ref_unpack(ans, b, int(t4[0]), chunk)
        resets = ev[ev[:, 0] == 1, 1].astype(np.uint32)
        _, rl, rk, rsts = O.ref_assemble_scans_ts(rnodes, rts, resets, MAX_NODES, MAX_SCANS)
        el, ests = _restated(O, ans, b, t4, rx[np.arange(len(b)) // chunk])
        assert rk == len(el) >= 3, (rk, len(el))
        assert (rl[:rk] == el).all()
        assert (rsts[:rk] == ests).all(), (ans, chunk, np.flatnonzero(rsts[:rk] != ests)[:5])
