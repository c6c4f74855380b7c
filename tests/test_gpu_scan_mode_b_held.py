"""GPU parity of LaserScan Mode B at stride 32768 against the CPU oracle, bit for bit, at every chunk count the two-CTA
cluster kernel (scan_tma.cu, scan_tma_cluster_kernel) can be given.

That kernel stages 1024-node chunk c in slot c >> 1 of CTA c & 1.  It keeps the chunks of the first kHeld slots in
registers and hands those slots back to its producer right after the mark pass; the other slots stay in shared memory
until the place pass.  The cases here do not depend on kHeld:

  * every chunk count from 1 to 32, each with the tail chunk full, one node short and one node over
    (1024 c - 1, 1024 c, 1024 c + 1), so that the boundary between held and resident slots, and the partial tail
    chunk, fall in either CTA on either side of that boundary;
  * duplicate measured keys between chunk 0 or 1 (held) and the scan's last chunk (resident unless the scan is short):
    once in the same CTA and once across the CTAs, at several lengths.  They go to the general kernel, and every
    slot must still be handed back exactly once: a slot handed back twice or not at all would stall the cluster's
    next scans, which follow in the same batch;
  * scans with nothing measured at lengths that end in a held and in a resident slot.

Each batch holds more scans than twice the 132 SMs of an H100, in a seeded shuffled order, so every cluster runs the
hand-back cycle over many scans of different lengths.  The case builder is checked without a GPU."""
import numpy as np
import pytest

from test_gpu_scan_parity import check_batch

CH = 1024
STRIDE = 32768
ROUNDS = 3
SM_COUNT = 132  # H100 SXM


def _chunk_counts():
    return [n for c in range(1, STRIDE // CH + 1) for n in (CH * c - 1, CH * c, CH * c + 1) if n <= STRIDE]


# (scan length, node of chunk 0 or 1, last node of the scan): the two nodes share a measured key
DUP_LENGTHS = (STRIDE, 17 * CH + 1, 18 * CH + 1, 9 * CH + 1)
NOTHING_LENGTHS = (9 * CH + 1, 17 * CH + 1, 24 * CH - 1)


def make_batch(oracle, seed):
    """One shuffled round: (nodes [scans, STRIDE], counts, expected path per scan, duplicate pairs (scan, i, j))."""
    rows, counts, paths, dups = [], [], [], []

    def add(nodes, n, path=0):
        row = np.zeros(STRIDE, oracle.NODE_DTYPE)
        row[:n] = nodes[:n]
        rows.append(row)
        counts.append(n)
        paths.append(path)

    for i, n in enumerate(_chunk_counts()):
        add(oracle.synth_batch(seed + i, 1, n, i % 2)[0], n)
    for i, n in enumerate(DUP_LENGTHS):
        base = oracle.synth_batch(seed + 500 + i, 1, n, 1)[0]
        for first in (5, CH + 5):  # chunk 0 (CTA 0) and chunk 1 (CTA 1)
            dup = base.copy()
            last = n - 1
            dup["angle_z_q14"][last] = dup["angle_z_q14"][first]
            dup["dist_mm_q2"][[first, last]] = [4000, 8000]
            dups.append((len(rows), first, last))
            add(dup, n, 1)  # 1 = PATH_GENERAL
    for i, n in enumerate(NOTHING_LENGTHS):
        nothing = oracle.synth_batch(seed + 600 + i, 1, n, 0)[0]
        nothing["dist_mm_q2"][:] = 0
        add(nothing, n)
    order = np.random.default_rng(seed).permutation(len(rows))
    where = {int(old): new for new, old in enumerate(order)}
    return (np.stack(rows)[order], np.array(counts, np.uint32)[order], np.array(paths, np.uint32)[order],
            [(where[s], i, j) for s, i, j in dups])


def test_case_builder_covers_the_held_boundary(oracle):
    nodes, counts, paths, dups = make_batch(oracle, 11000)
    assert nodes.shape[0] * ROUNDS > 2 * SM_COUNT
    assert set(_chunk_counts()) <= set(counts.tolist()) and max(counts) == STRIDE
    # every chunk count, with the tail chunk in both CTAs
    nch = (counts.astype(np.int64) + CH - 1) // CH
    assert set(nch.tolist()) == set(range(1, STRIDE // CH + 1))
    # duplicates: chunk 0 or 1 against the last chunk, in the same CTA and across the CTAs
    kinds = set()
    for s, i, j in dups:
        row = nodes[s]
        assert paths[s] == 1 and j == counts[s] - 1
        assert row["angle_z_q14"][i] == row["angle_z_q14"][j] and row["dist_mm_q2"][i] and row["dist_mm_q2"][j]
        ci, cj = i // CH, j // CH
        assert ci in (0, 1) and cj == nch[s] - 1
        kinds.add((cj, (ci & 1) == (cj & 1)))
    assert {(31, True), (31, False)} <= kinds  # chunk 31: the last slot of CTA 1
    assert any(same for _, same in kinds) and any(not same for _, same in kinds)
    # nothing-measured scans, and the other scans measured and tie-free
    empty = [s for s in range(len(counts)) if counts[s] and not nodes[s]["dist_mm_q2"][: counts[s]].any()]
    assert len(empty) == len(NOTHING_LENGTHS)
    for s in range(len(counts)):
        if paths[s] == 0 and s not in empty:
            keys = nodes[s]["angle_z_q14"][: counts[s]][nodes[s]["dist_mm_q2"][: counts[s]] != 0]
            assert len(np.unique(keys)) == len(keys)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.mark.gpu
def test_mode_b_every_chunk_count_and_held_duplicates(R, oracle):
    parts = [make_batch(oracle, 11000 + 1000 * r) for r in range(ROUNDS)]
    nodes = np.concatenate([p[0] for p in parts])
    counts = np.concatenate([p[1] for p in parts])
    expect_path = np.concatenate([p[2] for p in parts])
    assert nodes.shape[0] > 2 * SM_COUNT
    ctx = R.Context(0, STRIDE, nodes.shape[0])
    try:
        for newp in (0, 1):
            for inv in (0, 1):
                for ascend in (0, 1):
                    check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, stable=True, emit=False,
                                expect_path=expect_path)
    finally:
        ctx.close()
