"""GPU parity of LaserScan Mode B at stride 32768 against the CPU oracle, bit for bit, over long runs of consecutive
scans of one cluster of the two-CTA cluster kernel (scan_tma.cu, scan_tma_cluster_kernel).

That kernel is software-pipelined over the scans of its cluster: it marks the next streamed scan while it places the
current one, and clears the byte map for it between the two.  Cluster k of C serves scans k, k + C, k + 2 C, ...,
so a batch of C x ROUNDS scans laid out as round-major rows gives every cluster a sequence of ROUNDS scans of its own.
The sequences here are windows of one cyclic de Bruijn sequence over the scan kinds below, so that every kind of
scan follows every kind, itself included:

  * a placed scan (17 chunks and one node), a full 32-chunk scan, a 1-chunk scan (the second CTA gets no chunk) and
    a 3-chunk scan (fewer chunks than held slots in both CTAs);
  * scans handed to the general kernel: a duplicate measured key between chunk 0 and the last chunk (the same CTA)
    and between chunk 1 and the last chunk (across the CTAs);
  * a scan with nothing measured, an empty scan (count 0) and an invalid one (count above the stride).  The last two
    are not streamed: the pipeline passes over them to the next streamed scan.

Some clusters end on a short, an empty and an invalid scan, so the pipeline drains after each; a batch with fewer
scans than clusters runs each scan alone in its cluster.  C is the SM count over two, as the library sizes its grid;
on a GPU with another cluster count the parity checks still hold, only the pairs meant here would be others.  The
case builder is checked without a GPU."""
import numpy as np
import pytest

from helpers import bits
from test_gpu_scan_parity import check_batch, oracle_batch

CH = 1024
STRIDE = 32768
ROUNDS = 21
H100_CLUSTERS = 66  # 132 SMs of an H100 SXM, two per cluster

KINDS = ("placed", "full", "one_chunk", "three_chunk", "dup_same", "dup_across", "nothing", "empty", "invalid")
LENGTH = {"placed": 17 * CH + 1, "full": STRIDE, "one_chunk": 700, "three_chunk": 2 * CH + 500,
          "dup_same": 18 * CH + 1, "dup_across": 18 * CH + 1, "nothing": 9 * CH + 1, "empty": 0,
          "invalid": STRIDE + 1}
# cluster k's last scan: a short one, and two the kernel does not stream
LAST = {0: "one_chunk", 1: "three_chunk", 2: "empty", 3: "invalid"}


def de_bruijn(k):
    """Cyclic sequence of length k * k over 0..k-1 in which every ordered pair (a, b) appears once as neighbours."""
    a = [0] * (2 * k)
    seq = []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)

    db(1, 1)
    return seq


def cluster_kinds(clusters, rounds):
    """kinds[k][i]: the kind of cluster k's i-th scan."""
    cyc = [KINDS[i] for i in de_bruijn(len(KINDS))]
    out = []
    for k in range(clusters):
        off = (4 * k) % len(cyc)
        seq = [cyc[(off + i) % len(cyc)] for i in range(rounds)]
        if k in LAST:
            seq[-1] = LAST[k]
        out.append(seq)
    return out


def make_scan(oracle, kind, seed):
    """(row [STRIDE], count, expected path, duplicate pair or None)"""
    n = LENGTH[kind]
    if kind in ("empty", "invalid"):
        row = oracle.synth_batch(seed, 1, STRIDE, 1)[0]  # what a non-streamed scan's row holds is never read
        return row, n, 0, None
    row = oracle.synth_batch(seed, 1, n, seed % 2, stride=STRIDE)[0]
    if kind == "nothing":
        row["dist_mm_q2"][:n] = 0
    dup = None
    if kind in ("dup_same", "dup_across"):
        first, last = (5 if kind == "dup_same" else CH + 5), n - 1
        row["angle_z_q14"][last] = row["angle_z_q14"][first]
        row["dist_mm_q2"][[first, last]] = [4000, 8000]
        dup = (first, last)
    return row, n, (1 if dup else 0), dup


def make_batch(oracle, clusters, rounds, seed):
    """Round-major rows: scan i * clusters + k is cluster k's i-th.  Returns (nodes, counts, paths, kinds, dups)."""
    kinds = cluster_kinds(clusters, rounds)
    rows, counts, paths, flat, dups = [], [], [], [], {}
    for i in range(rounds):
        for k in range(clusters):
            kind = kinds[k][i]
            row, n, path, dup = make_scan(oracle, kind, seed + len(rows))
            if dup:
                dups[len(rows)] = dup
            rows.append(row)
            counts.append(n)
            paths.append(path)
            flat.append(kind)
    return np.stack(rows), np.array(counts, np.uint32), np.array(paths, np.uint32), flat, dups


def test_case_builder_covers_every_pair_of_consecutive_scans(oracle):
    assert len(de_bruijn(len(KINDS))) == len(KINDS) ** 2
    C = H100_CLUSTERS
    nodes, counts, paths, kinds, dups = make_batch(oracle, C, ROUNDS, 31000)
    assert nodes.shape == (C * ROUNDS, STRIDE) and ROUNDS >= 20
    pairs = set()
    for k in range(C):
        seq = [kinds[i * C + k] for i in range(ROUNDS)]
        pairs |= set(zip(seq, seq[1:]))
    assert pairs == {(a, b) for a in KINDS for b in KINDS}
    last = {kinds[(ROUNDS - 1) * C + k] for k in range(C)}
    assert {"one_chunk", "three_chunk", "empty", "invalid"} <= last
    for s, kind in enumerate(kinds):
        n = int(counts[s])
        assert n == LENGTH[kind] and (n > STRIDE) == (kind == "invalid")
        nch = -(-min(n, STRIDE) // CH)
        if kind == "one_chunk":
            assert nch == 1  # chunk 0 only: CTA 1 gets none
        if kind == "three_chunk":
            assert nch == 3  # two chunks in CTA 0, one in CTA 1: fewer than the held slots
        if kind == "nothing":
            assert n and not nodes[s]["dist_mm_q2"][:n].any()
        if kind in ("dup_same", "dup_across"):
            i, j = dups[s]
            assert paths[s] == 1 and j == n - 1 and j // CH == nch - 1
            assert nodes[s]["angle_z_q14"][i] == nodes[s]["angle_z_q14"][j]
            assert nodes[s]["dist_mm_q2"][i] and nodes[s]["dist_mm_q2"][j]
            assert ((i // CH) & 1 == (j // CH) & 1) == (kind == "dup_same")
        elif kind in ("placed", "full", "one_chunk", "three_chunk"):
            measured = nodes[s]["dist_mm_q2"][:n] != 0
            keys = nodes[s]["angle_z_q14"][:n][measured]
            assert measured.any() and len(np.unique(keys)) == len(keys) and paths[s] == 0


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _clusters():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count // 2


def check_batch_dev(R, oracle, ctx, nodes, counts, paths, newp, inv, ascend):
    """rpl_scan_batch_dev (counts on the device, so a count above the stride reaches the kernel) against the oracle
    bit for bit; the oracle sees the invalid scans as empty, and the kernel must report them and write nothing."""
    import torch

    S = nodes.shape[0]
    invalid = counts > STRIDE
    exp = oracle_batch(oracle, nodes, np.where(invalid, 0, counts).astype(np.uint32), newp, 0, inv, ascend)
    dev = torch.device("cuda")
    d_nodes = torch.from_numpy(nodes.view(np.uint8).reshape(S, STRIDE, 8)).to(dev)
    d_counts = torch.from_numpy(counts.astype(np.int32)).to(dev)
    ranges = torch.full((S, STRIDE), float("nan"), dtype=torch.float32, device=dev)
    intens = torch.full((S, STRIDE), float("nan"), dtype=torch.float32, device=dev)
    beams = torch.empty(S, dtype=torch.int32, device=dev)
    inc = torch.empty(S, dtype=torch.float32, device=dev)
    status = torch.empty(S, dtype=torch.int32, device=dev)
    path = torch.empty(S, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.scan_batch_dev(d_nodes.data_ptr(), d_counts.data_ptr(), S, STRIDE, R.scan_params(newp, 0, inv, ascend),
                       ranges=ranges.data_ptr(), intensities=intens.data_ptr(), beam_counts=beams.data_ptr(),
                       angle_increment=inc.data_ptr(), status=status.data_ptr(), path=path.data_ptr())
    ctx.synchronize()
    got_r, got_i = ranges.cpu().numpy(), intens.cpu().numpy()
    got_b = beams.cpu().numpy().view(np.uint32)
    got_inc, got_st = inc.cpu().numpy(), status.cpu().numpy().view(np.uint32)
    got_p = path.cpu().numpy().view(np.uint32)
    tag = (newp, inv, ascend)
    for s in range(S):
        if invalid[s]:
            assert got_st[s] == R.RESULT_INVALID_DATA and got_b[s] == 0 and bits(got_inc[s:s + 1])[0] == 0, (tag, s)
            assert got_p[s] == 0 and np.isnan(got_r[s]).all() and np.isnan(got_i[s]).all(), (tag, s)
            continue
        m = int(exp["beam_counts"][s])
        assert got_b[s] == m and got_st[s] == exp["status"][s] and got_p[s] == paths[s], (tag, s)
        assert bits(got_inc[s:s + 1])[0] == bits(exp["angle_increment"][s:s + 1])[0], (tag, s)
        assert (bits(got_r[s, :m]) == bits(exp["ranges"][s, :m])).all(), (tag, s)
        assert (bits(got_i[s, :m]) == bits(exp["intensities"][s, :m])).all(), (tag, s)


@pytest.mark.gpu
def test_mode_b_pipeline_every_pair_of_consecutive_scans(R, oracle):
    C = _clusters()
    nodes, counts, paths, _, _ = make_batch(oracle, C, ROUNDS, 31000)
    ctx = R.Context(0, STRIDE, nodes.shape[0])
    try:
        for newp, inv, ascend in ((0, 0, 1), (1, 1, 0), (0, 1, 1)):
            check_batch_dev(R, oracle, ctx, nodes, counts, paths, newp, inv, ascend)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_mode_b_pipeline_batch_smaller_than_the_clusters(R, oracle):
    """One scan per cluster: each is marked with nothing placed before it, and placed with nothing marked after it."""
    kinds = [k for k in KINDS if k != "invalid"]
    assert len(kinds) < _clusters()
    scans = [make_scan(oracle, kind, 32000 + i) for i, kind in enumerate(kinds)]
    nodes = np.stack([sc[0] for sc in scans])
    counts = np.array([sc[1] for sc in scans], np.uint32)
    paths = np.array([sc[2] for sc in scans], np.uint32)
    ctx = R.Context(0, STRIDE, len(kinds))
    try:
        for newp in (0, 1):
            for inv in (0, 1):
                for ascend in (0, 1):
                    check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, stable=True, emit=False,
                                expect_path=paths)
    finally:
        ctx.close()
