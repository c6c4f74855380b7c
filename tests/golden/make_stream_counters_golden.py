"""Generates tests/golden/stream_counters_golden.npz from the COMPILED REFERENCE (oracle/_ref).

Run where oracle/_ref is built (needs RPLIDAR_REFERENCE_DIR, a reference checkout):

    python tests/golden/make_stream_counters_golden.py

For every answer type (0x81..0x86) and seed of tests/test_stream_counters_pieces.py (GOLDEN_SEEDS):
  <ans>_<seed>_sha256  the SHA-256 of the damaged raw stream (T.golden_stream rebuilds it from the seed)
  <ans>_<seed>_events  (nodes, checksum errors, encoder resets, scan resets) of the SDK's unpacker fed it 7 bytes at a
                       time (the counts do not depend on the pieces: the test checks every piece size against it)
  <ans>_<seed>_lens    node count of every scan the SDK's ScanDataHolder (capacity GOLDEN_MAX_NODES) published
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import pyoracle as O  # noqa: E402

import test_stream_counters_pieces as T  # noqa: E402


def main():
    O.build(ref=True)
    assert O.have_ref() and O.have_ref_holder(), "the compiled reference (oracle/_ref) is needed"
    out = {}
    for ans in T.ALL_TYPES:
        for seed in T.GOLDEN_SEEDS:
            key = f"{ans:02x}_{seed}"
            b = T.golden_stream(O, ans, seed)
            events, rn, ev = T.sdk_events(O, ans, b, 7)
            _, rl, rk = O.ref_assemble_scans(rn, ev[ev[:, 0] == 1, 1].astype(np.uint32), T.GOLDEN_MAX_NODES, 4096)
            assert rk <= 4096
            out[f"{key}_sha256"] = np.frombuffer(T.stream_digest(b), np.uint8)
            out[f"{key}_events"] = np.array(events, np.int64)
            out[f"{key}_lens"] = rl[:rk].astype(np.uint32)
    np.savez_compressed(os.path.join(HERE, "stream_counters_golden.npz"), **out)


if __name__ == "__main__":
    main()
