"""GPU parity of LaserScan Mode B at strides above what the shared-memory kernels serve (32768 and 20000 nodes)
against the CPU oracle, bit for bit.  These scans run on the two-CTA cluster kernel (scan_tma.cu,
scan_tma_cluster_kernel), which stages 1024-node chunk c in CTA c & 1; the other tests only run full-length scans
here.  Covered: ragged counts around the chunk edges (0, 1, 1023 ... 32768), so that one CTA gets one chunk more
than the other or none at all; a scan with nothing measured; an unmeasured tail; and duplicate measured keys in
chunks 0 and 1 (across the two CTAs) and in chunks 0 and 2 (within one CTA), both of which must go to the general
kernel.  The batches hold more scans than an H100 has SMs, twice over, so every cluster runs several scans of
different lengths and reuses its slots and exchange barriers."""
import numpy as np
import pytest

from test_gpu_scan_parity import check_batch

pytestmark = pytest.mark.gpu

CH = 1024
ROUNDS = 19  # 19 x 15 scans: more than the 132 SMs of an H100, twice over


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 32768, 16 * ROUNDS)
    yield c
    c.close()


def _batch(oracle, stride, seed):
    """One round of cases at `stride`: (nodes, counts, expected path per scan)."""
    ragged = [n for n in (0, 1, 1023, 1024, 1025, 2049, 16383, 16385, 30001, 32767, 32768) if n <= stride]
    if stride not in ragged:
        ragged.append(stride)
    scans, counts, paths = [], [], []

    def add(nodes, n, path=0):
        row = np.zeros(stride, oracle.NODE_DTYPE)
        row[:n] = nodes[:n]
        scans.append(row)
        counts.append(n)
        paths.append(path)

    for i, n in enumerate(ragged):
        add(oracle.synth_batch(seed + i, 1, max(n, 1), i % 2)[0], n)
    full = oracle.synth_batch(seed + 100, 1, stride, 1)[0]
    nothing = full.copy()
    nothing["dist_mm_q2"][:] = 0                       # a scan with nothing measured
    add(nothing, stride)
    tail = full.copy()
    tail["dist_mm_q2"][stride - 3000:] = 0             # an unmeasured tail over the last chunks
    add(tail, stride)
    for j in (CH + 17, 2 * CH + 17):                   # chunk 1 (the other CTA) / chunk 2 (the same CTA as chunk 0)
        dup = full.copy()
        dup["angle_z_q14"][j] = dup["angle_z_q14"][5]  # a measured node of chunk 0 shares its key
        dup["dist_mm_q2"][[5, j]] = [4000, 8000]
        add(dup, stride, 1)                            # 1 = PATH_GENERAL
    return scans, counts, paths


@pytest.mark.parametrize("stride", [32768, 20000])
def test_mode_b_large_scans_ragged_and_duplicates(R, oracle, ctx, stride):
    scans, counts, paths = [], [], []
    for r in range(ROUNDS):
        s, c, p = _batch(oracle, stride, 7000 + 1000 * r)
        scans += s
        counts += c
        paths += p
    nodes = np.stack(scans)
    counts = np.array(counts, np.uint32)
    expect_path = np.array(paths, np.uint32)
    assert (expect_path == R.PATH_GENERAL).sum() == 2 * ROUNDS
    for newp in (0, 1):
        for inv in (0, 1):
            for ascend in (0, 1):
                check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, stable=True, emit=False,
                            expect_path=expect_path)
