"""The definition of the session nodes (rpl_*_stream_nodes*), pinned on the CPU: what RealLidarDriver::grab_scan_data
returns for a scan -- the holder's scan, capped by the holder first, then run through ascendScanData
(src/lidar_driver_wrapper.cpp:307-342) -- is oracle/scan_oracle.cpp's ascend (O.ascend) on the scans the restatement
publishes from the whole stream.  The GPU test (tests/test_gpu_stream_nodes.py) holds the sessions to the latter.

For streams of every answer type the SDK's own unpacker is fed the bytes in pieces, its own ScanDataHolder publishes
the scans and its own ascendScanData ascends each (oracle/_ref), return value included; where the compiled reference is
not built, the outputs it gave when tests/golden/stream_nodes_golden.npz was recorded stand in for it
(tests/golden/make_stream_nodes_golden.py).  Tie-free revolutions are compared bit for bit.  Where final keys tie, the
SDK's std::sort leaves the order among equal keys unspecified and the library follows its own stable rule: there the
key sequence and the set of nodes are compared."""
import os

import numpy as np
import pytest

from test_capsule_oracle_vs_ref import make_capsules
from test_capsule_stream_pieces import hq_capsules, restated_scans as capsule_restated
from test_decode_oracle_vs_ref import make_stream
from test_normal_stream_pieces import normal_stream, restated_scans as normal_restated

FAIL = 0x80008001
MAX_SCANS = 64
# name: (answer type, max_nodes of the holder); revolutions of about 650 nodes (ultra-dense: 2880), so 512 caps every
# one of them
CASES = {"express": (0x82, 2048), "hq": (0x83, 2048), "ultra": (0x84, 512), "dense": (0x85, 2048),
         "ultra_dense": (0x86, 512), "normal": (0x81, 2048), "normal_capped": (0x81, 512), "crafted": (0x83, 256)}


def crafted(O):
    """HQ capsules of hand-made revolutions with distinct keys: ordinary ones, one without a measured node, one of a
    single unmeasured node, and two longer than the holder's 256 nodes"""
    rng = np.random.default_rng(11)
    revs = []
    for n, measured in ((10, True), (120, True), (40, False), (300, True), (1, False), (33, True), (400, True), (2, True)):
        r = np.zeros(n, O.NODE_DTYPE)
        r["angle_z_q14"] = np.sort(rng.choice(65536, n, replace=False))
        r["dist_mm_q2"] = rng.integers(1, 160000, n) if measured else 0
        if measured:
            r["dist_mm_q2"][rng.random(n) < 0.15] = 0
            r["dist_mm_q2"][min(n - 1, 3)] = 4321
        r["quality"] = rng.integers(0, 256, n)
        r["flag"] = 2
        r["flag"][0] = 1
        revs.append(r)
    nodes = np.concatenate(revs + [revs[0][:1]])
    n = (len(nodes) + 95) // 96
    pad = np.zeros(n * 96 - len(nodes), O.NODE_DTYPE)
    pad["angle_z_q14"], pad["dist_mm_q2"], pad["flag"] = 7, 400, 2
    payload = np.zeros((n, 781), np.uint8)
    payload[:, 9:9 + 768] = np.concatenate([nodes, pad]).view(np.uint8).reshape(n, 768)
    return O.seal_capsules(0x83, payload)


def stream_of(O, name):
    """the case's wire bytes (flat uint8)"""
    ans = CASES[name][0]
    if name == "crafted":
        return crafted(O).reshape(-1)
    if ans == 0x81:
        return normal_stream(3300, 5, nodes_per_rev=650, bad=False)
    if ans == 0x83:
        return hq_capsules(O, 36, seed=4, nodes_per_rev=650).reshape(-1)
    if ans == 0x85:
        return make_stream(O, 90, 16.3, seed=3).reshape(-1)
    if ans == 0x86:  # (its decoder drops capsules whose start angles lie further apart: revolutions of 2880 nodes)
        return make_capsules(O, ans, 200, 45.0, seed=ans).reshape(-1)
    per = {0x82: 32, 0x84: 96}[ans]
    return make_capsules(O, ans, 3300 // per, 650.0 / per, seed=ans).reshape(-1)


def restated(O, name, b):
    ans, max_nodes = CASES[name]
    if ans == 0x81:
        return normal_restated(O, b, max_nodes, MAX_SCANS)[:3]
    return capsule_restated(O, ans, b.reshape(-1, O.capsule_bytes(ans)), max_nodes, MAX_SCANS)[:3]


def reference_grabs(O, name, b, chunk):
    """[(return value, nodes)] of the SDK fed `b` in pieces of `chunk` bytes (0: whole): unpacker, holder,
    ascendScanData"""
    ans, max_nodes = CASES[name]
    rn, ev = O.ref_unpack(ans, b, 31, chunk)
    resets = None if ans == 0x81 else ev[ev[:, 0] == 1, 1].astype(np.uint32)
    rs, rl, rk = O.ref_assemble_scans(rn, resets, max_nodes, MAX_SCANS)
    return [O.ref_ascend(rs[k, : rl[k]]) for k in range(min(rk, MAX_SCANS))]


def tie_free(buf):
    return len(np.unique(buf["angle_z_q14"])) == len(buf)


def check(O, name, grabs, b):
    """the grabs against O.ascend on the restated scans of the whole stream; returns the scans compared bit for bit"""
    es, el, ek = restated(O, name, b)
    assert len(grabs) == min(ek, MAX_SCANS) and ek >= 3
    exact = 0
    for k, (rc, buf) in enumerate(grabs):
        h = es[k, : el[k]]
        assert len(buf) == el[k] <= CASES[name][1], (name, k)  # the holder caps before the grab ascends
        erc, ebuf = O.ascend(h, stable=True)
        if (h["dist_mm_q2"] == 0).all():
            assert erc == FAIL and (ebuf.view(np.uint64) == h.view(np.uint64)).all()  # buffer unchanged
        assert rc == erc, (name, k)
        got, exp = np.ascontiguousarray(buf).view(np.uint64), ebuf.view(np.uint64)
        if tie_free(ebuf):
            exact += 1
            assert (got == exp).all(), (name, k)
        else:
            assert (buf["angle_z_q14"] == ebuf["angle_z_q14"]).all() and (np.sort(got) == np.sort(exp)).all(), (name, k)
    return exact


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_nodes_golden.npz")


@pytest.mark.parametrize("name", sorted(CASES))
def test_recorded_reference_grabs(oracle, name):
    """from the fixture alone: the recorded wire bytes and the reference's recorded grabs of them"""
    O = oracle
    g = np.load(GOLDEN)
    b, lens, rcs, nodes = g[f"{name}_bytes"], g[f"{name}_lens"], g[f"{name}_rc"], g[f"{name}_nodes"].view(O.NODE_DTYPE)
    ends = np.cumsum(lens)
    grabs = [(int(rcs[k]), nodes[ends[k] - lens[k]: ends[k]]) for k in range(len(lens))]
    exact = check(O, name, grabs, b)
    if name == "crafted":
        assert exact == len(lens)
        assert sorted(lens.tolist()) == [1, 2, 10, 33, 40, 120, 256, 256] and (rcs == FAIL).sum() == 2
    if CASES[name][1] == 512:
        assert (lens == 512).sum() >= 2  # revolutions longer than the holder: capped, then ascended


@pytest.mark.parametrize("chunk", [1, 7, 133, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_sdk_fed_in_pieces_then_ascended(oracle, name, chunk):
    O = oracle
    if not (O.have_ref() and O.have_ref_holder()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    b = stream_of(O, name)
    assert (b == np.load(GOLDEN)[f"{name}_bytes"]).all(), "the fixture was recorded from other bytes: regenerate it"
    check(O, name, reference_grabs(O, name, b, chunk), b)
