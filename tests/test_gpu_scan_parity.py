"""GPU parity tests proper (-m gpu): the CUDA path, called through the C-ABI, against the
CPU oracle on the same inputs.  Integer / index work must be bit-exact; the only floats on
this path (dist_m, intensity, angle_increment) are single correctly-rounded operations and
are compared bit-for-bit too."""
import numpy as np
import pytest

from helpers import bits

pytestmark = pytest.mark.gpu

ALL_MODES = [(newp, mode_a, inv) for newp in (0, 1) for mode_a in (0, 1) for inv in (0, 1)]


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 70000, 64)
    yield c
    c.close()


def _nodes(a, O):
    return np.ascontiguousarray(a).view(O.NODE_DTYPE).reshape(a.shape[:-1])


def oracle_batch(O, nodes, counts, newp, mode_a, inv, ascend, stable=True):
    buf = nodes.copy()
    prm = O.scan_params(newp, mode_a, inv, ascend, 40.0, 0.1)
    res = O.pipeline_batch(buf, counts, prm, stable=stable, threads=4)
    res["nodes"] = buf
    return res


def check_batch(R, O, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=0, stable=True, expect_path=None,
                emit=True):
    """rpl_scan_batch on the host arrays against the oracle, bit for bit.  Which kernel serves the batch is decided
    by rpl_capi.cu pick_fast; tests/test_gpu_scan_bands.py states the rule (DISPATCH) and asserts it case by
    case: flags & 1 the general kernel alone; stride <= 8192 and not flags & 4 the shared-memory kernels
    (scan_small.cu); else the ascended buffer (emit and ascend), flags & 2 or an odd stride scan_fast.cu; else Mode B
    at strides up to 32768 the two-CTA cluster kernel and everything else the TMA ring (scan_tma.cu).  The general
    kernel runs after every one of them for the scans they hand on (`path` 1)."""
    counts = np.asarray(counts, dtype=np.uint32)
    exp = oracle_batch(O, nodes, counts, newp, mode_a, inv, ascend, stable)
    got = ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts, R.scan_params(newp, mode_a, inv, ascend, flags),
                         emit_nodes=emit)
    if not emit:
        got["nodes"] = exp["nodes"]
    tag = (newp, mode_a, inv, ascend, flags, emit)
    assert (got["beam_counts"] == exp["beam_counts"]).all(), tag
    assert (got["status"] == exp["status"]).all(), tag
    assert (bits(got["angle_increment"]) == bits(exp["angle_increment"])).all(), tag
    for s in range(nodes.shape[0]):
        m, n = int(exp["beam_counts"][s]), int(counts[s])
        assert (bits(got["ranges"][s, :m]) == bits(exp["ranges"][s, :m])).all(), (tag, s)
        assert (bits(got["intensities"][s, :m]) == bits(exp["intensities"][s, :m])).all(), (tag, s)
        assert (got["nodes"][s, :n].view(np.uint64) == exp["nodes"][s, :n].view(np.uint64)).all(), (tag, s)
    if expect_path is not None:
        assert (got["path"] == expect_path).all(), (tag, got["path"])
    return got


# ---- config 1: A1 single scan, golden vectors from the compiled reference ------------------
@pytest.mark.parametrize("flags", [0, 1, 2])
def test_a1_golden_laserscan_bit_exact(R, oracle, ctx, golden_dir, flags):
    g = np.load(f"{golden_dir}/laserscan_golden.npz")
    d = np.load(f"{golden_dir}/dummy_scans.npz")
    var = _nodes(d["variants"], oracle)
    asc = _nodes(d["variants_ascended"], oracle)
    for k in range(int(g["n"])):
        vi, use_asc, newp, mode_a, inv = g[f"cfg_{k}"].tolist()
        res = ctx.scan(var[vi].view(R.NODE_DTYPE), R.scan_params(newp, mode_a, inv, use_asc, flags))
        assert res["beam_count"] == int(g[f"beams_{k}"]), k
        assert (bits(res["ranges"]) == bits(g[f"ranges_{k}"])).all(), k
        assert (bits(res["intensities"]) == bits(g[f"intens_{k}"])).all(), k
        assert bits(res["angle_increment"]) == bits(g[f"hdr_{k}"][2]), k
        if use_asc:
            assert res["ascend_status"] == int(d["variants_rc"][vi])
            assert (res["nodes"].view(np.uint64) == asc[vi].view(np.uint64)).all(), k
        else:
            assert (res["nodes"].view(np.uint64) == var[vi].view(np.uint64)).all(), k


def test_a1_all_sixteen_dummy_scans(R, oracle, ctx, golden_dir):
    d = np.load(f"{golden_dir}/dummy_scans.npz")
    raw = _nodes(d["raw"], oracle)
    counts = np.full(16, 360, np.uint32)
    for newp, mode_a, inv in ALL_MODES:
        check_batch(R, oracle, ctx, raw, counts, newp, mode_a, inv, 1, expect_path=0)


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_ascend_edge_cases_golden(R, oracle, ctx, golden_dir, flags):
    g = np.load(f"{golden_dir}/ascend_cases.npz")
    for i in range(int(g["n_cases"])):
        inp = _nodes(g[f"in_{i}"], oracle)
        if flags == 0:
            rc, out = ctx.ascend_scan(inp.view(R.NODE_DTYPE))  # TMA kernel when aligned
        else:
            r = ctx.scan(inp.view(R.NODE_DTYPE), R.scan_params(0, 0, 0, 1, flags))
            rc, out = r["ascend_status"], r["nodes"]
        assert rc == int(g[f"rc_{i}"]), i
        assert (out.view(np.uint8).reshape(-1, 8) == g[f"out_{i}"]).all(), i
    rc, out = ctx.ascend_scan(oracle.make_nodes([3, 2, 1], [0, 0, 0]).view(R.NODE_DTYPE))
    assert rc == R.RESULT_OPERATION_FAIL and out["angle_z_q14"].tolist() == [3, 2, 1]
    rc, _ = ctx.ascend_scan(np.zeros(0, R.NODE_DTYPE))
    assert rc == R.RESULT_OPERATION_FAIL
    r, i, m, inc = ctx.laserscan(np.zeros(0, R.NODE_DTYPE), R.scan_params())
    assert m == 0


# ---- synthetic scans (SURVEY.md 8(d)) --------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 17, 360, 3200, 8192, 32768])
@pytest.mark.parametrize("variant", [0, 1, 3])
def test_tie_free_synthetic_both_kernels(R, oracle, ctx, n, variant):
    nodes = oracle.synth_batch(5000 + 10 * variant + n, 5, n, variant)
    counts = np.full(5, n, np.uint32)
    modes = ALL_MODES if n in (360, 3200) else [(0, 0, 0), (1, 1, 0), (0, 1, 1), (1, 0, 1)]
    for newp, mode_a, inv in modes:
        for ascend in (0, 1):
            # tie-free measured keys: the reference's std::sort and the stable rule coincide
            for flags in ((0, 2, 4, 6) if n <= 8192 else (0, 2)):
                for emit in (True, False):
                    # (with the ascended buffer a fill key may collide with a measured key: that scan then takes
                    # the general kernel, legitimately -- so the path is only pinned without it)
                    check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=flags, stable=True,
                                emit=emit, expect_path=None if emit else 0)
            check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=1, stable=True,
                        expect_path=1)


@pytest.mark.parametrize("n", [2, 64, 2048, 32768])
def test_tie_variant_follows_stable_rule(R, oracle, ctx, n):
    nodes = oracle.synth_batch(900 + n, 4, n, 2)
    counts = np.full(4, n, np.uint32)
    for newp, mode_a, inv in [(0, 0, 0), (0, 1, 0), (1, 1, 1), (1, 0, 1)]:
        for ascend in (0, 1):
            for flags in (0, 2, 4, 6):
                check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=flags, stable=True)
            check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, stable=True, emit=False)
    # the reference itself (unstable sort) agrees wherever order is defined: Mode A ranges
    exp = oracle_batch(oracle, nodes, counts, 0, 1, 0, 1, stable=False)
    got = ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts, R.scan_params(0, 1, 0, 1))
    for s in range(4):
        m = int(exp["beam_counts"][s])
        assert (bits(got["ranges"][s, :m]) == bits(exp["ranges"][s, :m])).all()


def test_mixed_batch_ragged_counts_and_paths(R, oracle, ctx):
    """One batch mixing tie-free and tie scans, empty scans, all-unmeasured scans, odd counts
    and a stride larger than every count."""
    stride = 1000
    rng = np.random.default_rng(3)
    counts = np.array([0, 1, 999, 360, 513, 7, 1000, 64, 250, 2], np.uint32)
    nodes = np.zeros((len(counts), stride), oracle.NODE_DTYPE)
    for s, n in enumerate(counts):
        if n == 0:
            continue
        variant = [0, 2, 3, 1][s % 4]
        nodes[s, :n] = oracle.synth_batch(40 + s, 1, int(n), variant)[0]
    nodes[3]["dist_mm_q2"][:] = 0  # a scan with no measurement at all
    nodes[6]["dist_mm_q2"][: 37] = 0  # long unmeasured head (serial head tune)
    nodes[8]["angle_z_q14"][:] = rng.integers(0, 8, size=stride)  # heavy ties
    for newp, mode_a, inv in ALL_MODES:
        for ascend in (0, 1):
            got = check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend)
            for flags in (2, 4, 6):
                check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=flags)
            for flags in (0, 4):
                check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=flags, emit=False)
    assert got["status"][3] == R.RESULT_OPERATION_FAIL and got["beam_counts"][3] == 0
    assert got["path"][8] == R.PATH_GENERAL


def test_extreme_values(R, oracle, ctx):
    """dist_mm_q2 up to 2^32-1 (float rounding collisions in dist_m), keys 0 and 65535, a bin
    shared by many points, more than 65536 nodes (cannot be tie-free)."""
    mk = oracle.make_nodes
    n = 4096
    keys = np.arange(n) * 16
    keys[-1] = 65535
    dist = np.full(n, 0xFFFFFFFF, np.uint64)
    dist[::3] = 0xFFFFFF00
    dist[::5] = 1
    a = mk(keys, dist, np.arange(n) % 256)
    narrow = mk(np.arange(1000), np.random.default_rng(1).integers(1, 9000, 1000), np.arange(1000) % 256)
    nodes = np.zeros((2, n), oracle.NODE_DTYPE)
    nodes[0] = a
    nodes[1, :1000] = narrow
    counts = np.array([n, 1000], np.uint32)
    for newp, mode_a, inv in ALL_MODES:
        check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 1)
        check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 1, emit=False)
        check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 1, flags=4, emit=False)
        check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 1, flags=6)
        check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 0, flags=1)
    big = oracle.synth_batch(1, 1, 70000, 0)
    check_batch(R, oracle, ctx, big, np.array([70000], np.uint32), 0, 1, 0, 1, expect_path=1)
    check_batch(R, oracle, ctx, big, np.array([70000], np.uint32), 1, 0, 1, 1, expect_path=1)


def test_invalid_arguments_fail_loudly(R, ctx):
    nodes = np.zeros((1, 8), R.NODE_DTYPE)
    with pytest.raises(R.RplError):
        ctx.scan_batch(nodes, np.array([9], np.uint32), R.scan_params())  # count > stride
    with pytest.raises(R.RplError):
        big = np.zeros((65, 8), R.NODE_DTYPE)
        ctx.scan_batch(big, np.full(65, 8, np.uint32), R.scan_params())  # n_scans > max_scans


# ---- synthetic generator and full-size properties ---------------------------------------------
@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4])
def test_device_synth_equals_oracle_synth(R, oracle, ctx, variant):
    import torch

    for n in (1, 7, 360, 3200, 32768):
        t = torch.zeros((3, n, 8), dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(3, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
        ctx.synth_batch_dev(11 + variant, 3, n, n, variant, t.data_ptr(), cnt.data_ptr())
        ctx.synchronize()
        torch.cuda.synchronize()
        exp = oracle.synth_batch(11 + variant, 3, n, variant)
        assert (t.cpu().numpy().reshape(3, n, 8) == exp.view(np.uint8).reshape(3, n, 8)).all(), (variant, n)
        assert (cnt.cpu().numpy() == n).all()


def test_full_size_batch_properties(R, oracle):
    """BASELINE.json configs[1] at full size (4096 x 32768): size-independent properties checked
    on the device with torch as an independent checker, plus oracle parity on sampled scans."""
    import torch

    S, N = 4096, 32768
    ctx = R.Context(0, N, S)
    dev = torch.device("cuda")
    nodes = torch.empty((S, N, 8), dtype=torch.uint8, device=dev)
    counts = torch.empty(S, dtype=torch.int32, device=dev)
    ranges = torch.full((S, N), float("nan"), dtype=torch.float32, device=dev)
    intens = torch.full((S, N), float("nan"), dtype=torch.float32, device=dev)
    beams = torch.empty(S, dtype=torch.int32, device=dev)
    inc = torch.empty(S, dtype=torch.float32, device=dev)
    status = torch.empty(S, dtype=torch.int32, device=dev)
    path = torch.empty(S, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.synth_batch_dev(0, S, N, N, 1, nodes.data_ptr(), counts.data_ptr())
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.scan_batch_dev(nodes.data_ptr(), counts.data_ptr(), S, N, R.scan_params(0, 0, 0, 1), ranges=ranges.data_ptr(),
                       intensities=intens.data_ptr(), beam_counts=beams.data_ptr(), angle_increment=inc.data_ptr(),
                       status=status.data_ptr(), path=path.data_ptr())
    ctx.synchronize()
    torch.cuda.synchronize()
    assert int((path != 0).sum()) == 0 and int((status != 0).sum()) == 0
    w = nodes.view(torch.int32).reshape(S, N, 2)
    x, y = w[..., 0], w[..., 1]
    key = (x & 0xFFFF).to(torch.int32)
    dist = ((x >> 16) & 0xFFFF) | ((y & 0xFFFF) << 16)
    qual = (y >> 16) & 0xFF
    valid = dist != 0
    assert (valid.sum(1).to(torch.int32) == beams).all()
    chunk = 512
    for s0 in range(0, S, chunk):
        sl = slice(s0, s0 + chunk)
        # unmeasured nodes sort to the end: key + 65536
        k2 = torch.where(valid[sl], key[sl], key[sl] + 65536)
        order = torch.argsort(k2, dim=1, stable=True)
        # divide by a CUDA tensor: `tensor / python_scalar` multiplies by the reciprocal in torch
        four_k = torch.full((1, 1), 4000.0, dtype=torch.float32, device=dev)
        d_sorted = torch.gather(dist[sl], 1, order).to(torch.float32) / four_k
        q_sorted = (torch.gather(qual[sl], 1, order) >> 2).to(torch.float32)
        m = beams[sl].to(torch.int64)
        live = torch.arange(N, device=dev)[None, :] < m[:, None]
        assert torch.equal(ranges[sl][live].view(torch.int32), d_sorted[live].view(torch.int32))
        assert torch.equal(intens[sl][live].view(torch.int32), q_sorted[live].view(torch.int32))
        assert bool(torch.isnan(ranges[sl][~live]).all())  # nothing written past beam_count
    # oracle parity on sampled scans
    for s in (0, 1, 2047, 4095):
        host = nodes[s].cpu().numpy().view(oracle.NODE_DTYPE).reshape(1, N)
        exp = oracle.pipeline_batch(host.copy(), np.array([N], np.uint32), oracle.scan_params(0, 0, 0, 1, 40.0, 0.1))
        m = int(exp["beam_counts"][0])
        assert m == int(beams[s])
        assert (ranges[s, :m].cpu().numpy().view(np.uint32) == exp["ranges"][0, :m].view(np.uint32)).all()
        assert bits(inc[s:s + 1].cpu().numpy())[0] == bits(exp["angle_increment"])[0]
    ctx.close()


def test_odd_stride_takes_unaligned_path(R, oracle, ctx):
    """An odd stride puts every second scan on an 8-byte (not 16-byte) boundary: the library must
    fall back from the TMA kernel to the register-streamed kernel, with identical results."""
    stride, n = 1001, 997
    nodes = np.zeros((6, stride), oracle.NODE_DTYPE)
    nodes[:, :n] = oracle.synth_batch(321, 6, n, 1)
    counts = np.full(6, n, np.uint32)
    for newp, mode_a, inv in ALL_MODES:
        for flags in (0, 4):  # shared-memory kernel without TMA staging / register-streamed kernel
            for emit in (True, False):
                check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, 1, flags=flags, emit=emit,
                            expect_path=None if emit else 0)


def test_mode_a_sorted_revolution_detection_edge_cases(R, oracle, ctx):
    """Mode A on shapes that stress the order-dependent parts of its kernels (the TMA kernel's index map and run
    detection, the shared-memory kernels' per-bin minimum): sorted / rotated / two interleaved ascending runs (one
    descent, but not a rotation) / unmeasured runs across chunk boundaries (1024 nodes) and around the wrap / bins
    shared by many points and long empty stretches."""
    rng = np.random.default_rng(77)
    n = 12288
    cases = []
    base_keys = np.sort(rng.choice(65536, size=n, replace=False))
    dist = rng.integers(600, 160000, n)
    q = rng.integers(0, 256, n)
    cases.append(oracle.make_nodes(base_keys, dist, q, 2))                                   # sorted
    cases.append(np.roll(cases[0], -5000))                                                   # rotated
    inter = cases[0].copy()
    half = n // 2
    inter["angle_z_q14"][:half] = base_keys[0::2]
    inter["angle_z_q14"][half:] = base_keys[1::2]
    cases.append(inter)                                                                      # one descent, no rotation
    gaps = np.roll(cases[0], -1021).copy()
    gaps["dist_mm_q2"][1000:1100] = 0     # unmeasured run across the first chunk boundary
    gaps["dist_mm_q2"][n - 30:] = 0       # ... at the end of the buffer
    gaps["dist_mm_q2"][:17] = 0           # ... and at its start
    gaps["dist_mm_q2"][n - 1021 - 3: n - 1021 + 3] = 0  # around the wrap of the rotation
    cases.append(gaps)
    dense = cases[0].copy()
    dense["angle_z_q14"] = np.sort(np.concatenate([rng.choice(np.arange(20000, 20600), 500, replace=False),
                                                   rng.choice(np.arange(40000, 65536), n - 500, replace=False)]))
    cases.append(np.roll(dense, -777))                                                       # crowded bins + a long gap
    nodes = np.stack(cases)
    counts = np.full(len(cases), n, np.uint32)
    for newp, inv in ((0, 0), (1, 1), (1, 0)):
        check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, 1, emit=False, expect_path=0)
        check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, 0, emit=False, expect_path=0)
    small = nodes[:, :8000].copy()  # the same shapes through the TMA kernel at a size the shared-memory kernels serve
    check_batch(R, oracle, ctx, small, np.full(len(cases), 8000, np.uint32), 0, 1, 0, 1, flags=4, emit=False)
    check_batch(R, oracle, ctx, small, np.full(len(cases), 8000, np.uint32), 0, 1, 0, 1, flags=0, emit=False)


def test_mode_a_duplicate_keys_in_the_shared_memory_kernel(R, oracle, ctx):
    """Mode A without the ascended buffer keeps no bitmap of the keys: a scan with duplicate keys stays on the
    shared-memory kernel unless two points with the SAME key hold a bin's minimum dist_m with DIFFERENT qualities
    (only then does the order among equal keys matter: the stable rule takes the first in buffer order).  Each of
    the cases, checked against the oracle's stable rule, with the path each must take."""
    rng = np.random.default_rng(5)
    n = 3000
    keys = np.sort(rng.choice(65536, size=n, replace=False))
    dist = rng.integers(4000, 160000, n)
    q = rng.integers(0, 256, n)
    base = oracle.make_nodes(keys, dist, q, 2)

    def with_dup(i, j, dist_j, q_j):  # node j gets node i's key
        c = base.copy()
        c["angle_z_q14"][j] = c["angle_z_q14"][i]
        c["dist_mm_q2"][j] = dist_j
        c["quality"][j] = q_j
        return c

    d100 = int(base["dist_mm_q2"][100])
    q100 = int(base["quality"][100])
    harmless = [
        with_dup(100, 2000, d100 + 4000, q100 ^ 0x40),   # same key, the duplicate is farther: it never wins
        with_dup(100, 2000, d100, q100),                 # same key, same distance, same quality: indistinguishable
        with_dup(100, 50, d100 - 400, q100 ^ 0x40),      # the duplicate (earlier in the buffer) is nearer: it wins on distance
    ]
    conflicts = [
        with_dup(100, 2000, d100, q100 ^ 0x40),          # same key, same distance, other quality, later in the buffer
        with_dup(100, 50, d100, q100 ^ 0x40),            # ... earlier in the buffer: the duplicate is the first
    ]
    # make sure the duplicated key really holds its bin's minimum in the conflict cases (nothing nearer in the bin)
    for c in conflicts + harmless:
        c["dist_mm_q2"][99] = max(int(c["dist_mm_q2"][99]), d100 + 8000)
        c["dist_mm_q2"][101] = max(int(c["dist_mm_q2"][101]), d100 + 8000)
    for group, path in ((harmless, 0), (conflicts, R.PATH_GENERAL)):
        nodes = np.stack(group)
        counts = np.full(len(group), n, np.uint32)
        for newp, inv in ((0, 0), (1, 1)):
            for ascend in (0, 1):
                check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, emit=False, stable=True, expect_path=path)
                check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, emit=True, stable=True)
                check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, flags=4, emit=False, stable=True)
    # heavy duplication: every key four times with random distances and qualities
    heavy = oracle.make_nodes(np.repeat(keys[: n // 4], 4), rng.integers(4000, 4100, n), rng.integers(0, 4, n) * 64, 2)
    heavy = heavy[rng.permutation(n)]
    for newp, inv in ((0, 0), (1, 1)):
        check_batch(R, oracle, ctx, heavy[None], np.array([n], np.uint32), newp, 1, inv, 1, emit=False, stable=True)


def test_shared_final_keys_are_resolved_in_the_shared_memory_kernel(R, oracle, ctx):
    """With the ascended buffer, the interpolated key of an unmeasured node can land on a measured node's key.  Up
    to 16 such nodes per revolution are placed by the shared-memory kernel itself (stable rule: equal keys in buffer
    order), more go to the general kernel.  Tie-free synthetic revolutions of 3200 nodes with 5 % unmeasured nodes:
    the ones where that happens (a few per cent) must stay on the fast path and match the oracle bit for bit; then
    hand-made cases: a key shared by three nodes, 16 and 17 shared keys."""
    n = 3200
    pool = oracle.synth_batch(424242, 1500, n, 0)
    counts = np.full(pool.shape[0], n, np.uint32)
    exp = oracle_batch(oracle, pool, counts, 0, 0, 0, 1, True)
    keys = exp["nodes"]["angle_z_q14"]
    shared = np.flatnonzero((np.diff(keys.astype(np.int32), axis=1) == 0).any(axis=1))
    assert len(shared) >= 10, len(shared)  # the situation the bench meets in ~4 % of its revolutions
    sel = pool[shared[:64]]
    for newp, mode_a, inv in ((0, 0, 0), (1, 1, 1), (0, 1, 0), (1, 0, 1)):
        check_batch(R, oracle, ctx, sel, np.full(len(sel), n, np.uint32), newp, mode_a, inv, 1, emit=True, expect_path=0)
    # hand-made: measured keys 100, 200, ... ; unmeasured nodes get their keys from the fill, so put MEASURED
    # duplicates next to them in Mode A (which keeps no bitmap of the measured keys) to reach exact counts
    rng = np.random.default_rng(12)
    base_keys = np.sort(rng.choice(np.arange(64, 65000), size=2000, replace=False))
    for n_shared, path in ((1, 0), (3, 0), (16, 0), (17, R.PATH_GENERAL)):
        k = base_keys.copy()
        # n_shared extra nodes: the first three on ONE key (a key held by up to four nodes), the rest on distinct keys
        src = np.concatenate([np.full(min(n_shared, 3), 500), 600 + 7 * np.arange(max(n_shared - 3, 0))]).astype(int)
        dst = 1500 + 3 * np.arange(n_shared)
        k[dst] = k[src]
        dist = rng.integers(4000, 160000, len(k))
        c = oracle.make_nodes(k, dist, rng.integers(0, 256, len(k)), 2)
        c = c[rng.permutation(len(c))]
        for newp, inv in ((0, 0), (1, 1)):
            check_batch(R, oracle, ctx, c[None], np.array([len(c)], np.uint32), newp, 1, inv, 1, emit=True, stable=True,
                        expect_path=path)
            check_batch(R, oracle, ctx, c[None], np.array([len(c)], np.uint32), newp, 0, inv, 1, emit=True, stable=True,
                        expect_path=R.PATH_GENERAL)  # Mode B ranks the measured keys: any duplicate among them


def test_mode_b_duplicate_measured_keys_in_the_shared_memory_kernel(R, oracle, ctx):
    """Mode B without the ascended buffer: up to 16 measured nodes beyond the first of their key are placed by the
    shared-memory kernel itself (stable rule: equal keys in buffer order), more go to the general kernel.  The pattern
    the capsule -> LaserScan chain produces (first and last node of a revolution on one key), a key held by four
    nodes, unmeasured nodes on a shared key (they do not count), exactly 16 and 17."""
    rng = np.random.default_rng(21)
    n = 3201
    keys = np.sort(rng.choice(np.arange(8, 65500), size=n, replace=False))
    dist = rng.integers(4000, 160000, n)
    q = rng.integers(0, 256, n)

    def make(n_shared, unmeasured_twin=False):
        k = keys.copy()
        if n_shared == 1:
            k[-1] = k[0]                       # first and last node of the revolution meet
        else:
            src = np.concatenate([np.full(min(n_shared, 3), 700), 900 + 5 * np.arange(max(n_shared - 3, 0))]).astype(int)
            k[2000 + 3 * np.arange(n_shared)] = k[src]
        c = oracle.make_nodes(k, dist, q, 2)
        if unmeasured_twin:
            c["dist_mm_q2"][1234] = 0
            c["angle_z_q14"][1234] = c["angle_z_q14"][50]   # an unmeasured node on a measured node's key: no duplicate
        return c

    for n_shared, path in ((1, 0), (3, 0), (16, 0), (17, R.PATH_GENERAL)):
        for twin in (False, True):
            c = make(n_shared, twin)
            for rot in (0, 1500):
                scan = np.roll(c, -rot)[None]
                for newp, inv in ((0, 0), (1, 1)):
                    for ascend in (0, 1):
                        check_batch(R, oracle, ctx, scan, np.array([n], np.uint32), newp, 0, inv, ascend, emit=False,
                                    stable=True, expect_path=path)
                        check_batch(R, oracle, ctx, scan, np.array([n], np.uint32), newp, 0, inv, ascend, flags=4,
                                    emit=False, stable=True)
