"""The contract of the dense stream session, pinned on the CPU: the SDK's own unpacker fed a stream in pieces, then its
own ScanDataHolder, publishes exactly the scans the restatement (oracle/decode_oracle.cpp) publishes from the whole
stream in one call.  The session (rpl_capsule_stream_* on 0x85, tests/test_gpu_dense_stream.py) is held to the latter, so
this is what makes "any split into pushes gives the whole stream's scans" the SDK's behaviour and not a new definition.
Needs the compiled reference (oracle/_ref); skipped without it."""
import numpy as np
import pytest

from test_decode_oracle_vs_ref import make_stream


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_ref() and oracle.have_ref_holder()):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return oracle


def _prime(O):
    # the SDK keeps the last node's scan-start flag in a function-static: leave it at 0 (a short clean stretch whose
    # last node is no scan start), so that the streams here start fresh like the restatement
    O.ref_dense_decode(make_stream(O, 3, 80.0, seed=1, start_deg=100.0).reshape(-1), 31, 84)


def _stream(O, seed):
    rng = np.random.default_rng(seed)
    caps = make_stream(O, 600, 80.0 + (seed % 5), seed=seed, sync_every=290 + seed % 30)
    caps[rng.choice(600, 8, replace=False), 10] ^= 0x40  # checksum errors
    caps[rng.choice(600, 4, replace=False)] = 0          # bad frames
    caps[-1] = 0 if seed % 2 else caps[-1]
    return caps


@pytest.mark.parametrize("chunk", [1, 84, 84 * 3 + 7, 84 * 40, 84 * 81, 84 * 500])
def test_sdk_fed_in_pieces_publishes_the_whole_streams_scans(O, chunk):
    for seed in (11, 12, 13):
        caps = _stream(O, seed)
        _prime(O)
        rn, ev = O.ref_dense_decode(caps.reshape(-1), 31, chunk)
        rres = ev[ev[:, 0] == 1, 1].astype(np.uint32)
        rs, rl, rk = O.ref_assemble_scans(rn, rres, 2048, 64)
        en, es, eo, _ = O.dense_decode(caps, 31, 0)
        es_, el, ek = O.assemble_scans(en, O.resets_from_capsules(es, eo), 2048, 64)
        assert rk == ek and ek >= 3 and (rl == el).all()
        for k in range(min(ek, 64)):
            assert (rs[k, : rl[k]].view(np.uint64) == es_[k, : el[k]].view(np.uint64)).all(), (seed, chunk, k)
    _prime(O)
