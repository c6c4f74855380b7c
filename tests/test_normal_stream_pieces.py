"""The contract of the standard-node stream session (0x81), pinned on the CPU: the SDK's own unpacker
(UnpackerHandler_NormalNode) fed a raw byte stream in pieces, then its own ScanDataHolder, publishes exactly the scans
the restatement (oracle decode_normal + the holder restatement) publishes from the whole stream in one call.  The session
(rpl_capsule_stream_*_bytes on 0x81, tests/test_gpu_normal_stream.py) is held to the latter, so this is what makes "any
split of the bytes into pushes gives the whole stream's scans" the SDK's behaviour for 0x81 and not a new definition
(tests/test_capsule_stream_pieces.py does the same for the capsule formats).  Needs the compiled reference (oracle/_ref);
skipped without it.

The stream builder here is shared with the GPU test."""
import numpy as np
import pytest

NODES_PER_REV = 3200  # records per revolution (the dense format's 80 x 40)


def normal_stream(n_records, seed, nodes_per_rev=NODES_PER_REV, bad=True, noise=200):
    """one 0x81 byte stream of revolutions: angles rise through each revolution, whose first record carries the sync
    bit.  With `bad`: records whose check bit or sync-bit pair fails, dropped and inserted bytes, and a stretch of
    `noise` random bytes, all of which send the byte machine hunting for the next record."""
    rng = np.random.default_rng(seed)
    pos = (np.arange(n_records) + int(rng.integers(0, nodes_per_rev))) % nodes_per_rev
    start = (pos == 0).astype(np.uint8)
    rec = np.zeros((n_records, 5), np.uint8)
    rec[:, 0] = (rng.integers(0, 64, n_records).astype(np.uint8) << 2) | ((1 - start) << 1) | start
    q6 = (pos * (360 * 64) // nodes_per_rev + rng.integers(0, 3, n_records)) % (360 * 64)
    w = (q6 << 1) | 1  # the check bit
    rec[:, 1], rec[:, 2] = w & 0xFF, w >> 8
    dist = rng.integers(0, 65536, n_records)
    dist[rng.random(n_records) < 0.05] = 0
    rec[:, 3], rec[:, 4] = dist & 0xFF, dist >> 8
    b = rec.reshape(-1)
    if not bad:
        return b
    k = max(2, n_records // 4000)
    idx = rng.choice(n_records, k, replace=False)
    b[5 * idx[: k // 2] + 1] &= 0xFE  # check bit cleared
    b[5 * idx[k // 2:]] ^= 0x01       # sync bit equal to its inverse
    b = np.delete(b, rng.choice(len(b), k, replace=False))
    b = np.insert(b, np.sort(rng.choice(len(b), k, replace=False)), rng.integers(0, 256, k).astype(np.uint8))
    at = int(rng.integers(0, len(b)))
    return np.concatenate([b[:at], rng.integers(0, 256, noise, dtype=np.uint8), b[at:]])


def restated_scans(O, b, max_nodes, max_scans=512):
    """(scans, lengths, published, nodes, fsm_pos): the restatement's decoder and holder on the whole stream (the
    standard unpacker requests no scan resets)"""
    nodes, _, pos = O.decode_normal(b)
    s, l, k = O.assemble_scans(nodes, None, max_nodes, max_scans)
    return s, l, k, nodes, pos


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_ref() and oracle.have_ref_holder()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle


def _streams():
    out = [normal_stream(20000, seed) for seed in (31, 32)]
    out.append(normal_stream(16000, 33, bad=False)[:-3])  # a clean stream ending inside a record
    return out


@pytest.mark.parametrize("max_nodes", [2048, 4096])
@pytest.mark.parametrize("chunk", [1, 2, 3, 4, 5, 6, 7, 64, 0])  # 0: the whole stream in one call
def test_sdk_fed_in_pieces_publishes_the_whole_streams_scans(O, chunk, max_nodes):
    max_scans = 128
    for i, b in enumerate(_streams()):
        rn, ev = O.ref_unpack(0x81, b, 31, chunk)
        assert not (ev[:, 0] == 1).any()  # no scan-reset requests from the standard unpacker
        rs, rl, rk = O.ref_assemble_scans(rn, None, max_nodes, max_scans)
        es, el, ek, nodes, _ = restated_scans(O, b, max_nodes, max_scans)
        assert len(rn) == len(nodes) and (rn.view(np.uint64) == nodes.view(np.uint64)).all()
        assert rk == ek and ek >= 3 and (rl == el).all()
        for k in range(min(ek, max_scans)):
            assert (rs[k, : rl[k]].view(np.uint64) == es[k, : el[k]].view(np.uint64)).all(), (chunk, k)
        # the clean stream's revolutions of 3200 records: the holder's capacity rule cuts them at 2048
        assert i < 2 or (el[:ek] == min(max_nodes, NODES_PER_REV)).all()
