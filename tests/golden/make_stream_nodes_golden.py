"""Generates tests/golden/stream_nodes_golden.npz from the COMPILED REFERENCE (oracle/_ref).

Run where oracle/_ref is built (needs RPLIDAR_REFERENCE_DIR, a reference checkout):

    python tests/golden/make_stream_nodes_golden.py

For every case of tests/test_stream_nodes_pieces.py:
  <case>_bytes   the wire bytes of the stream (uint8)
  <case>_lens    node count of every scan the SDK's ScanDataHolder published, the unpacker fed 7 bytes at a time
  <case>_rc      the SDK's ascendScanData return value for each of them
  <case>_nodes   their nodes after ascendScanData, one behind the other (uint64 per node)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import pyoracle as O  # noqa: E402

import test_stream_nodes_pieces as T  # noqa: E402


def main():
    O.build(ref=True)
    assert O.have_ref() and O.have_ref_holder(), "the compiled reference (oracle/_ref) is needed"
    out = {}
    for name in sorted(T.CASES):
        b = T.stream_of(O, name)
        grabs = T.reference_grabs(O, name, b, 7)
        T.check(O, name, grabs, b)
        out[f"{name}_bytes"] = b
        out[f"{name}_lens"] = np.array([len(n) for _, n in grabs], np.uint32)
        out[f"{name}_rc"] = np.array([rc for rc, _ in grabs], np.uint32)
        out[f"{name}_nodes"] = np.concatenate([np.ascontiguousarray(n).view(np.uint64) for _, n in grabs])
    np.savez_compressed(os.path.join(HERE, "stream_nodes_golden.npz"), **out)


if __name__ == "__main__":
    main()
