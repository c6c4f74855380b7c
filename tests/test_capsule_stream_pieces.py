"""The contract of the capsule stream session for express (0x82), HQ (0x83), ultra (0x84) and ultra-dense (0x86)
capsules, pinned on the CPU: the SDK's own unpacker fed a stream in byte pieces, then its own ScanDataHolder, publishes
exactly the scans the restatement (oracle/capsule_oracle.cpp + the holder restatement) publishes from the whole stream
in one call.  The session (rpl_capsule_stream_*, tests/test_gpu_capsule_stream.py) is held to the latter, so this is
what makes "any split into pushes gives the whole stream's scans" the SDK's behaviour for these formats and not a new
definition (tests/test_dense_stream_pieces.py does the same for dense capsules).  Needs the compiled reference
(oracle/_ref); skipped without it.

The stream builders here are shared with the GPU test."""
import numpy as np
import pytest

from test_capsule_oracle_vs_ref import make_capsules

STREAM_FORMATS = [0x82, 0x83, 0x84, 0x86]
# capsules per revolution: about 2600-2900 nodes per revolution in every format (dense: 80 x 40 = 3200)
CAPS_PER_REV = {0x82: 80.0, 0x84: 30.0, 0x85: 80.0, 0x86: 45.0}
HQ_NODES_PER_REV = 2880


def hq_capsules(O, n, seed=0, nodes_per_rev=HQ_NODES_PER_REV):
    """HQ capsules carrying ordered revolutions: angles rise through each revolution, whose first node has flag bit 0
    set (random node flags would cut revolutions a few nodes long)."""
    rng = np.random.default_rng(seed)
    pos = (np.arange(n * 96) + int(rng.integers(0, nodes_per_rev))) % nodes_per_rev
    nodes = np.zeros(n * 96, O.NODE_DTYPE)
    nodes["angle_z_q14"] = (pos * 65536 // nodes_per_rev + rng.integers(0, 3, n * 96)) & 0xFFFF
    nodes["dist_mm_q2"] = rng.integers(0, 40000 * 4, n * 96)
    nodes["dist_mm_q2"][rng.random(n * 96) < 0.05] = 0
    nodes["quality"] = rng.integers(0, 256, n * 96)
    start = pos == 0
    nodes["flag"] = start.astype(np.uint8) | ((~start).astype(np.uint8) << 1)
    payload = rng.integers(0, 256, (n, 781), dtype=np.uint8)
    payload[:, 9:9 + 768] = nodes.view(np.uint8).reshape(n, 768)
    return O.seal_capsules(0x83, payload)


def format_stream(O, ans, n, seed, sync_every=None, bad=True, near=False):
    """[n, capsule bytes]: one stream of the format, with scan-start capsules every `sync_every` (not HQ: its scan
    starts are node flags), and with `bad` a few checksum / CRC errors and all-zero capsules"""
    if ans == 0x83:
        caps = hq_capsules(O, n, seed)
    else:
        caps = make_capsules(O, ans, n, CAPS_PER_REV[ans] + (seed % 7) * 0.3, seed=seed, sync_every=sync_every,
                             near=near)
    if bad:
        rng = np.random.default_rng(seed + 1)
        caps[rng.choice(n, max(1, n // 60), replace=False), 20] ^= 0x08  # checksum / CRC errors
        caps[rng.choice(n, max(1, n // 120), replace=False)] = 0          # bad frames (all zero)
    return caps


def restated_scans(O, ans, caps, max_nodes, max_scans=512):
    """(scans, lengths, published, nodes, status, offsets): the restatement's decoder and holder on the whole stream"""
    nodes, status, offs, _ = O.decode_capsules(ans, caps, 31)
    s, l, k = O.assemble_scans(nodes, O.resets_from_capsules(status, offs), max_nodes, max_scans)
    return s, l, k, nodes, status, offs


def _ref_pieces(O, ans, caps, chunk, max_nodes, max_scans):
    rn, ev = O.ref_unpack(ans, caps.reshape(-1), 31, chunk)
    return O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), max_nodes, max_scans)


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_ref() and oracle.have_ref_holder()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle


def _streams(O, ans):
    cb = O.capsule_bytes(ans)
    out = [format_stream(O, ans, 600, seed, sync_every=250 + seed) for seed in (21, 22)]
    clean = format_stream(O, ans, 500, 23, bad=False)
    clean[-1] = 0  # a stream ending on an all-zero capsule
    out.append(clean)
    if ans == 0x86:
        out += [format_stream(O, ans, 300, seed, sync_every=130, near=True) for seed in (24, 25)]
    assert all(c.shape[1] == cb for c in out)
    return out


@pytest.mark.parametrize("ans", STREAM_FORMATS)
@pytest.mark.parametrize("piece", ["1", "7", "cb-1", "cb+1", "3cb+7", "whole"])
def test_sdk_fed_in_pieces_publishes_the_whole_streams_scans(O, ans, piece):
    cb = O.capsule_bytes(ans)
    chunk = {"1": 1, "7": 7, "cb-1": cb - 1, "cb+1": cb + 1, "3cb+7": 3 * cb + 7, "whole": 0}[piece]
    max_nodes, max_scans = 2048, 64
    for i, caps in enumerate(_streams(O, ans)):
        rs, rl, rk = _ref_pieces(O, ans, caps, chunk, max_nodes, max_scans)
        es, el, ek, nodes, status, _ = restated_scans(O, ans, caps, max_nodes, max_scans)
        assert rk == ek and ek >= 3 and (rl == el).all()
        for k in range(min(ek, max_scans)):
            assert (rs[k, : rl[k]].view(np.uint64) == es[k, : el[k]].view(np.uint64)).all(), (ans, chunk, k)
        if i < 2:  # the streams with errors and (but HQ) scan-start capsules
            assert (status & O.CAPSULE_CHECKSUM_ERR).any()
            assert ans == 0x83 or (status & O.CAPSULE_SYNC).any()
