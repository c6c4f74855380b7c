"""The scan kernels across their whole size range, against the CPU oracle (stable rule) bit for bit, with the kernel
that ran made visible.

pick_fast (rpl_capi.cu) picks one of five kernels per launch from the stride, the base alignment, the mode, the
ascended buffer and the flags, for batches and single scans alike (a single scan is a batch of one at the context's
stride: max_nodes rounded up to even).  Every kernel hands a scan it cannot serve to scan_general_kernel, so a change to the dispatch leaves every result correct and
moves a test case onto a different kernel without any parity test noticing.  Here each case runs under the CUDA
profiler and asserts the kernel it expects (kernels_run, DISPATCH), then covers what the other tests never reach:

  * the 32769..65536-node band, device-resident, with more scans than the ring grid so that every persistent CTA's
    ring wraps inside a scan and across scan boundaries (test_band_*);
  * the full key space: 65536 nodes, every key once (M = 65536, inverted Mode B writes from slot 65535), its
    one-duplicate twin and 65537 nodes (test_full_key_space);
  * the ring kernel's Mode A index map at its limit, M = 32768 (served) and 32769 (handed on), with measured nodes up
    to buffer index 65535 (test_mode_a_index_map_limit);
  * the single-scan entry points at real sizes, in a context much larger than the scan and in one exactly its size
    (test_single_scan_at_real_sizes);
  * PointCloud2 above the shared-memory kernels and the float64 projection of the every-key scan (test_cloud_*).

The case builders are checked without a GPU (test_case_builders_make_what_the_gpu_tests_rely_on)."""
import os
import re
import time

import numpy as np
import pytest

from helpers import bits
from test_gpu_cloud import check_cloud, room_scans
from test_gpu_scan_parity import ALL_MODES, check_batch

gpu = pytest.mark.gpu

THREADS = max(1, min(os.cpu_count() or 1, 16))  # oracle worker threads

# short kernel names (what kernels_run reports)
SMALL = "scan_small_kernel"
CLUSTER = "scan_tma_cluster_kernel"
RING_B, RING_A, RING_CLOUD = "scan_tma_kernel<0>", "scan_tma_kernel<1>", "scan_tma_kernel<2>"
FAST_B, FAST_A = "scan_fast_kernel<false,false>", "scan_fast_kernel<false,true>"
FAST_EMIT_B, FAST_EMIT_A = "scan_fast_kernel<true,false>", "scan_fast_kernel<true,true>"
GENERAL = "scan_general_kernel"
SOR, VOXEL = "cloud_sor_kernel", "cloud_voxel_kernel"

KEYS = 65536               # angle_z_q14 is a u16: larger scans cannot be tie-free (kMaxFastNodes)
MODE_A_MAP_MAX = 32768     # scan_tma.cu kModeASmemMaxPoints: u-ranks the ring kernel's Mode A index map holds
CH = 1024                  # nodes per chunk of the TMA kernels
BAND_STRIDES = (32770, 40000, 49152, 65536)
BAND_COUNTS = (0, 1, 1023, 1025, 16383, 16384, 16385, 32767, 32769, 49153, 65535)
POOL = 19                  # distinct scans per band batch: prime, so CTAs of any grid meet every case in turn


# ---- which kernel ran ----------------------------------------------------------------------------------------------
_B = r"(?:\(bool\)\s*)?(true|false|1|0)"
_KERNEL_NAMES = (
    (re.compile(r"scan_tma_cluster_kernel"), lambda m: CLUSTER),
    (re.compile(r"scan_tma_kernel\s*<\s*(?:\(int\)\s*)?(\d)\s*>"), lambda m: f"scan_tma_kernel<{m[1]}>"),
    (re.compile(r"scan_tma_kernelILi(\d)E"), lambda m: f"scan_tma_kernel<{m[1]}>"),  # mangled
    (re.compile(r"scan_fast_kernel\s*<\s*" + _B + r"\s*,\s*" + _B + r"\s*>"),
     lambda m: "scan_fast_kernel<%s,%s>" % tuple("true" if v in ("true", "1") else "false" for v in (m[1], m[2]))),
    (re.compile(r"scan_fast_kernelILb([01])ELb([01])E"),
     lambda m: "scan_fast_kernel<%s,%s>" % tuple("true" if v == "1" else "false" for v in (m[1], m[2]))),
    (re.compile(r"scan_small_kernel"), lambda m: SMALL),
    (re.compile(r"scan_general_kernel"), lambda m: GENERAL),
    (re.compile(r"cloud_sor_kernel"), lambda m: SOR),
    (re.compile(r"cloud_voxel_kernel"), lambda m: VOXEL),
)
_OURS = re.compile(r"scan_(small|tma|fast|general)|cloud_(sor|voxel)_kernel")


def _short_name(name):
    for rx, short in _KERNEL_NAMES:
        m = rx.search(name)
        if m:
            return short(m)
    assert not _OURS.search(name), f"kernel name not recognised: {name!r}"
    return None


def kernels_run(fn, ctx) -> set:
    """Runs fn() under the CUDA profiler and returns the short names of the library's kernels that ran.  The library
    launches on its own streams in the primary context; CUPTI activity tracing records kernels from every stream."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx.synchronize()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # without a margin, the trace of a call launched right after the profiler started came back empty now and
        # then (the profiler keeps only activity inside its capture window): keep the kernels clear of both edges
        time.sleep(0.02)
        fn()
        ctx.synchronize()
        torch.cuda.synchronize()
        time.sleep(0.02)
    names = [e.name for e in prof.events()]
    raw = getattr(getattr(prof, "profiler", None), "kineto_results", None)
    if raw is not None:
        names += [e.name() for e in raw.events()]
    ran = {s for s in map(_short_name, names) if s}
    if not ran:
        print(f"kernels_run: the profiler recorded {len(names)} events, none of them the library's: {names[:8]}")
    return ran


# ---- case builders (plain numpy + the oracle's generator; checked on the CPU below) ---------------------------------
def measured_everywhere(nodes):
    """The same nodes with every unmeasured one given a distance: no fill keys, so no fill-key collisions."""
    out = nodes.copy()
    d = out["dist_mm_q2"]
    d[d == 0] = 4321
    return out


def tie_free(O, n, seed, variant=1):
    """One scan of n nodes, every node measured, keys distinct while n <= 65536."""
    return measured_everywhere(O.synth_batch(seed, 1, n, variant)[0])


def with_duplicate(scan, i=5, j=None):
    """Measured node j takes measured node i's key (a duplicated measured key)."""
    out = scan.copy()
    j = len(out) // 2 + 17 if j is None else j
    out["angle_z_q14"][j] = out["angle_z_q14"][i]
    out["dist_mm_q2"][[i, j]] = [4000, 8000]
    return out


def band_pool(O, stride, seed):
    """POOL scans of one band batch: (nodes [POOL, stride], counts, duplicate flag per scan).  Behind each count the
    row holds measured nodes whose keys collide with the live ones, so reading past the count cannot go unnoticed."""
    counts = sorted({min(c, stride) for c in BAND_COUNTS} | {stride})
    rows, cnt, dup = [], [], []

    def add(live, n, is_dup=False):
        row = measured_everywhere(O.synth_batch(seed + 977 + len(rows), 1, stride, 0)[0])
        row[:n] = live[:n]
        rows.append(row)
        cnt.append(n)
        dup.append(is_dup)

    for i, n in enumerate(counts):  # ragged counts at the chunk and ring edges
        add(O.synth_batch(seed + i, 1, max(n, 1), (0, 1, 3)[i % 3])[0], n)
    full = O.synth_batch(seed + 100, 1, stride, 1)[0]
    nothing = full.copy()
    nothing["dist_mm_q2"][:] = 0                   # nothing measured
    add(nothing, stride)
    tail = full.copy()
    tail["dist_mm_q2"][stride - 3 * CH - 17:] = 0  # an unmeasured tail over the last chunks
    add(tail, stride)
    last_chunk = (stride - 1) // CH
    add(with_duplicate(full, 5, min(40, last_chunk) * CH + (17 if 40 < last_chunk else 0)), stride, True)  # chunk 0/40
    k = 0
    while len(rows) < POOL:
        add(O.synth_batch(seed + 300 + k, 1, stride, (0, 1, 3)[k % 3])[0], stride)
        k += 1
    return np.stack(rows), np.array(cnt, np.uint32), np.array(dup)


def full_key_space(O, seed=4242):
    """65536 nodes, every key exactly once, every node measured, starting anywhere in the revolution."""
    s = measured_everywhere(O.synth_batch(seed, 1, KEYS, 0)[0])
    return np.roll(s, -12345)


def one_node_too_many(O):
    """65537 nodes: the whole key space measured once plus one unmeasured node -- no measured key repeats, the count
    alone exceeds what the fast kernels take."""
    full = full_key_space(O)
    extra = O.make_nodes([777], [0], [0], 2)
    return np.concatenate([full[:30000], extra, full[30000:]])


def mode_a_limit_scan(O, n, m, with_key0, seed):
    """n nodes of which exactly m are measured, on m distinct keys: a run of 20000 consecutive keys (Mode A bins of
    two and three points), keys 40000..51999 left empty (a long stretch of empty bins), the rest drawn at random; key 0
    measured or not.  The measured nodes sit at random buffer positions including the last one (index n - 1), in the
    order of a revolution that starts anywhere; the unmeasured ones carry random keys."""
    rng = np.random.default_rng(seed)
    lo = 0 if with_key0 else 1
    dense = np.arange(lo, lo + 20000)
    rest = np.setdiff1d(np.arange(lo + 20000, KEYS), np.arange(40000, 52000))
    keys = np.sort(np.concatenate([dense, rng.choice(rest, m - len(dense), replace=False)]))
    keys = np.roll(keys, -int(rng.integers(0, m)))
    pos = np.sort(np.concatenate([rng.choice(n - 1, m - 1, replace=False), [n - 1]]))
    out = O.make_nodes(rng.integers(0, KEYS, n), np.zeros(n, np.uint32), np.zeros(n, np.uint8), 2)
    out[pos] = O.make_nodes(keys, rng.integers(600, 160000, m), rng.integers(0, 256, m), 2)
    return out


def measured_keys(scan, n=None):
    live = scan[: len(scan) if n is None else n]
    return live["angle_z_q14"][live["dist_mm_q2"] != 0]


def has_duplicate(scan, n=None):
    k = measured_keys(scan, n)
    return len(np.unique(k)) != len(k)


# ---- comparisons ---------------------------------------------------------------------------------------------------
def oracle_scans(O, nodes, counts, newp, mode_a, inv, ascend):
    buf = nodes.copy()
    res = O.pipeline_batch(buf, counts, O.scan_params(newp, mode_a, inv, ascend, 40.0, 0.1), stable=True,
                           threads=THREADS)
    res["nodes"] = buf
    return res


def expected_path(kernel, scan, n):
    """1 where the fast kernels must hand the scan to the general kernel, else 0 (input without fill-key collisions)."""
    if kernel is None or n > KEYS or has_duplicate(scan, n):
        return 1
    return int(kernel == RING_A and len(measured_keys(scan, n)) > MODE_A_MAP_MAX)


def dev_batch(R, O, ctx, pool, counts, idx, newp, mode_a, inv, ascend, flags=0, emit=False, offset=0,
              expect_path=None, profile=False):
    """scan_batch_dev on the scans pool[idx] (one device buffer at `offset` bytes past a 512-byte boundary), compared
    with the oracle on the pool, on the device: ranges and intensities up to beam_count bit for bit and NaN (the
    pre-fill) behind it, beam_count, angle_increment, status, path where expect_path[p] >= 0, the ascended nodes when
    emitted.  Returns the kernels that ran when profile is set."""
    import torch

    dev = torch.device("cuda")
    P, stride = pool.shape
    S, nb = len(idx), stride * 8
    idx_t = torch.from_numpy(np.asarray(idx, np.int64)).to(dev)
    pool_t = torch.from_numpy(pool.view(np.uint8).reshape(P, nb)).to(dev)
    raw = torch.empty(S * nb + 16, dtype=torch.uint8, device=dev)
    nodes = raw[offset: offset + S * nb].view(S, nb)
    nodes.copy_(pool_t[idx_t])
    counts_t = torch.from_numpy(counts.astype(np.int32)).to(dev)[idx_t].contiguous()
    ranges = torch.full((S, stride), float("nan"), dtype=torch.float32, device=dev)
    intens = torch.full((S, stride), float("nan"), dtype=torch.float32, device=dev)
    beams, status, path = (torch.full((S,), -1, dtype=torch.int32, device=dev) for _ in range(3))
    inc = torch.full((S,), float("nan"), dtype=torch.float32, device=dev)
    nodes_out = nodes.clone() if emit else None  # the kernels write only the scans they ascend
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ptr = nodes.data_ptr()
    assert ptr % 16 == offset % 16

    def call():
        ctx.scan_batch_dev(ptr, counts_t.data_ptr(), S, stride, R.scan_params(newp, mode_a, inv, ascend, flags),
                           nodes_out=None if nodes_out is None else nodes_out.data_ptr(), ranges=ranges.data_ptr(),
                           intensities=intens.data_ptr(), beam_counts=beams.data_ptr(), angle_increment=inc.data_ptr(),
                           status=status.data_ptr(), path=path.data_ptr())
        ctx.synchronize()
        torch.cuda.synchronize()

    ran = kernels_run(call, ctx) if profile else call()
    tag = (stride, newp, mode_a, inv, ascend, flags, emit, offset)
    exp = oracle_scans(O, pool, counts, newp, mode_a, inv, ascend)
    idx = np.asarray(idx)
    got_b = beams.cpu().numpy().view(np.uint32)
    assert (got_b == exp["beam_counts"][idx]).all(), (tag, np.flatnonzero(got_b != exp["beam_counts"][idx])[:8])
    assert (status.cpu().numpy().view(np.uint32) == exp["status"][idx]).all(), tag
    assert (bits(inc.cpu().numpy()) == bits(exp["angle_increment"])[idx]).all(), tag
    if expect_path is not None:
        want = np.asarray(expect_path)[idx]
        got_p = path.cpu().numpy()
        pinned = want >= 0
        assert (got_p[pinned] == want[pinned]).all(), (tag, np.flatnonzero(got_p[pinned] != want[pinned])[:8])
    er = torch.from_numpy(exp["ranges"].view(np.int32)).to(dev)
    ei = torch.from_numpy(exp["intensities"].view(np.int32)).to(dev)
    en = torch.from_numpy(exp["nodes"].view(np.uint8).reshape(P, nb)).to(dev) if emit else None
    col = torch.arange(stride, device=dev)
    for c0 in range(0, S, 64):
        sl = slice(c0, min(S, c0 + 64))
        live = col[None, :] < beams[sl, None]
        for got, want in ((ranges[sl], er[idx_t[sl]]), (intens[sl], ei[idx_t[sl]])):
            ok = torch.where(live, got.view(torch.int32) == want, torch.isnan(got))
            if not bool(ok.all()):
                s = c0 + int((~ok).any(1).nonzero()[0])
                pytest.fail(f"{tag}: scan {s} (pool {idx[s]}, count {counts[idx[s]]}) differs from the oracle or was "
                            f"written past beam_count")
        if emit:
            ok = (nodes_out[sl] == en[idx_t[sl]]).all(1)
            assert bool(ok.all()), (tag, c0 + int((~ok).nonzero()[0]))
    del raw, nodes, nodes_out, ranges, intens, er, ei, en, pool_t
    return ran


def check_single(R, O, ctx, call, scan, newp, mode_a, inv, ascend, flags=0):
    """One scan through ctx.scan / ctx.laserscan / ctx.ascend_scan against the oracle."""
    n = len(scan)
    tag = (call, n, newp, mode_a, inv, ascend, flags, ctx.max_nodes)
    if call == "ascend_scan":
        rc, got = ctx.ascend_scan(scan.view(R.NODE_DTYPE))
        exp_rc, exp = O.ascend(scan, stable=True)
        assert rc == exp_rc, tag
        assert (got.view(np.uint64) == exp.view(np.uint64)).all(), tag
        return
    if call == "laserscan":
        ascend = 0
    exp = oracle_scans(O, scan[None], np.array([n], np.uint32), newp, mode_a, inv, ascend)
    m = int(exp["beam_counts"][0])
    prm = R.scan_params(newp, mode_a, inv, ascend, flags)
    if call == "laserscan":
        r, i, got_m, got_inc = ctx.laserscan(scan.view(R.NODE_DTYPE), prm)
    else:
        got = ctx.scan(scan.view(R.NODE_DTYPE), prm)
        r, i, got_m, got_inc = got["ranges"], got["intensities"], got["beam_count"], got["angle_increment"]
        assert got["ascend_status"] == int(exp["status"][0]), tag
        assert (got["nodes"].view(np.uint64) == exp["nodes"][0].view(np.uint64)).all(), tag
    assert got_m == m, (tag, got_m, m)
    assert bits(np.array([got_inc], np.float32))[0] == bits(exp["angle_increment"])[0], tag
    assert (bits(r) == bits(exp["ranges"][0, :m])).all(), tag
    assert (bits(i) == bits(exp["intensities"][0, :m])).all(), tag


# ---- A. the profiler sees the library's kernels --------------------------------------------------------------------
@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@gpu
def test_profiler_sees_the_library_kernels(R, oracle):
    with R.Context(0, 3200, 2) as ctx:
        nodes = oracle.synth_batch(1, 2, 3200, 0)
        ran = kernels_run(lambda: ctx.scan_batch(nodes.view(R.NODE_DTYPE), np.full(2, 3200, np.uint32),
                                                 R.scan_params(0, 0, 0, 1)), ctx)
    if not ran:
        pytest.fail("torch.profiler recorded none of the library's kernels: CUDA activity tracing (CUPTI) is not "
                    "available here, so no kernel assertion in this file can hold")
    assert ran == {SMALL, GENERAL}, ran


# ---- B. the dispatch table -----------------------------------------------------------------------------------------
NS, NT, FG = 4, 2, 1  # RPL_FLAG_NO_SMALL, RPL_FLAG_NO_TMA, RPL_FLAG_FORCE_GENERAL
# (entry, stride, count, base offset in bytes, mode_a, ascend, emit, flags, duplicate key) -> the fast kernel that
# must run (None: none, the general kernel serves every scan).  Batches (batch = rpl_scan_batch, dev =
# rpl_scan_batch_dev, status = rpl_scan_batch without LaserScan or ascended buffer, cloud = rpl_cloud_batch) run
# scan_general_kernel after it, always; single scans (scan, laserscan, ascend_scan; the count is given, the stride is
# the context's) run it only when a scan is handed on.  One rule for both: FORCE_GENERAL or nothing to produce ->
# general only; stride <= 8192 and not NO_SMALL -> shared-memory kernel; PointCloud2 with an unaligned base or odd
# stride -> general only; the ascended buffer (emit with ascend), NO_TMA (LaserScan only), an odd stride or a base not
# 16-byte aligned -> scan_fast_kernel; LaserScan Mode B at strides in (8192, 32768] -> the cluster kernel; else the
# ring kernel.  The single scans here run in a 70002-node context (stride 70002); SIZED_SINGLE below runs them in a
# context of their own size.
DISPATCH = [
    # stride <= 8192
    ("batch", 3200, 3200, 0, 0, 1, False, 0, False, SMALL),
    ("batch", 3200, 3200, 0, 1, 1, True, 0, False, SMALL),
    ("batch", 8192, 8191, 0, 0, 0, False, 0, False, SMALL),
    ("batch", 3200, 3200, 0, 0, 1, False, NS, False, RING_B),
    ("batch", 3200, 3200, 0, 1, 1, False, NS, False, RING_A),
    ("batch", 3200, 3200, 0, 0, 0, True, NS, False, RING_B),         # buffer passed through, no ascend: ring
    ("batch", 3200, 3200, 0, 0, 1, True, NS, False, FAST_EMIT_B),
    ("batch", 3200, 3200, 0, 1, 1, True, NS, False, FAST_EMIT_A),
    ("batch", 3201, 3201, 0, 0, 1, False, NS, False, FAST_B),
    ("batch", 3201, 3200, 0, 1, 0, False, NS, False, FAST_A),
    ("batch", 3200, 3200, 0, 0, 1, False, NS | NT, False, FAST_B),
    ("dev", 3200, 3200, 8, 0, 1, False, 0, False, SMALL),
    ("dev", 3200, 3200, 8, 0, 1, False, NS, False, FAST_B),
    # (8192, 32768]
    ("batch", 8194, 8194, 0, 0, 1, False, 0, False, CLUSTER),
    ("batch", 20000, 20000, 0, 0, 1, False, 0, False, CLUSTER),
    ("batch", 32768, 32768, 0, 0, 0, False, 0, False, CLUSTER),
    ("batch", 32768, 32768, 0, 0, 0, False, 0, True, CLUSTER),
    ("batch", 20000, 20000, 0, 0, 0, True, 0, False, CLUSTER),       # buffer passed through, no ascend
    ("batch", 32768, 32767, 0, 1, 1, False, 0, False, RING_A),
    ("batch", 20000, 20000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("batch", 20000, 20000, 0, 1, 1, True, 0, False, FAST_EMIT_A),
    ("batch", 20000, 20000, 0, 0, 1, False, NT, False, FAST_B),
    ("batch", 20000, 20000, 0, 1, 1, False, NT, False, FAST_A),
    ("batch", 8193, 8193, 0, 0, 1, False, 0, False, FAST_B),
    ("batch", 20001, 20001, 0, 1, 1, False, 0, False, FAST_A),
    ("dev", 20000, 20000, 8, 0, 1, False, 0, False, FAST_B),
    ("dev", 20000, 20000, 16, 0, 1, False, 0, False, CLUSTER),
    ("dev", 20000, 20000, 8, 1, 1, False, 0, False, FAST_A),
    ("dev", 20000, 20000, 16, 1, 1, False, 0, False, RING_A),
    # (32768, 65536]
    ("batch", 32770, 32770, 0, 0, 1, False, 0, False, RING_B),
    ("batch", 40000, 40000, 0, 0, 0, False, 0, False, RING_B),
    ("batch", 65536, 65536, 0, 0, 1, False, 0, False, RING_B),
    ("batch", 40000, 40000, 0, 0, 1, False, 0, True, RING_B),
    ("batch", 40000, 32000, 0, 1, 1, False, 0, False, RING_A),
    ("batch", 65536, 65536, 0, 1, 0, False, 0, False, RING_A),      # M > 32768: handed on
    ("batch", 40000, 40000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("batch", 65536, 65536, 0, 1, 1, True, 0, False, FAST_EMIT_A),
    ("batch", 40000, 40000, 0, 0, 0, True, 0, False, RING_B),        # buffer passed through, no ascend
    ("batch", 40000, 40000, 0, 0, 1, False, NT, False, FAST_B),
    ("batch", 65536, 65536, 0, 1, 1, False, NT, False, FAST_A),
    ("batch", 40001, 40001, 0, 0, 1, False, 0, False, FAST_B),
    ("batch", 65535, 65535, 0, 1, 1, False, 0, False, FAST_A),
    ("dev", 40000, 40000, 8, 0, 1, False, 0, False, FAST_B),
    ("dev", 40000, 40000, 16, 0, 1, False, 0, False, RING_B),
    ("dev", 40000, 32000, 8, 1, 1, False, 0, False, FAST_A),
    ("dev", 40000, 32000, 16, 1, 1, False, 0, False, RING_A),
    ("dev", 40000, 40000, 16, 0, 1, True, 0, False, FAST_EMIT_B),
    # > 65536: the fast kernels hand every scan on
    ("batch", 70000, 70000, 0, 0, 1, False, 0, False, RING_B),
    ("batch", 70000, 70000, 0, 1, 1, True, 0, False, FAST_EMIT_A),
    ("batch", 70001, 70001, 0, 0, 1, False, 0, False, FAST_B),
    # the general kernel alone
    ("batch", 3200, 3200, 0, 0, 1, False, FG, False, None),
    ("batch", 40000, 40000, 0, 1, 1, True, FG, False, None),
    ("status", 3200, 3200, 0, 0, 1, False, 0, False, None),
    ("status", 40000, 40000, 0, 0, 0, True, 0, False, None),        # buffer passed through, nothing else to produce
    # PointCloud2
    ("cloud", 3200, 3200, 0, 0, 0, False, 0, False, SMALL),
    ("cloud", 3200, 3200, 0, 0, 0, False, NS, False, RING_CLOUD),   # CLOUD_NO_FUSED
    ("cloud", 20000, 20000, 0, 0, 0, False, 0, False, RING_CLOUD),
    ("cloud", 40000, 40000, 0, 0, 0, False, 0, False, RING_CLOUD),
    ("cloud", 40001, 40001, 0, 0, 0, False, 0, False, None),
    # single scans
    ("laserscan", 360, 360, 0, 0, 0, False, 0, False, RING_B),
    ("laserscan", 3200, 3200, 0, 1, 0, False, 0, False, RING_A),
    ("laserscan", 40000, 40000, 0, 0, 0, False, 0, False, RING_B),
    ("laserscan", 40000, 40000, 0, 1, 0, False, 0, False, RING_A),   # M > 32768: handed on
    ("laserscan", 40000, 40000, 0, 1, 0, False, NT, False, FAST_A),
    ("laserscan", 70000, 70000, 0, 0, 0, False, 0, False, RING_B),   # > 65536: handed on
    ("scan", 360, 360, 0, 1, 0, False, 0, False, RING_A),
    ("scan", 3200, 3200, 0, 0, 0, False, 0, False, RING_B),
    ("scan", 40000, 40000, 0, 0, 0, False, 0, False, RING_B),
    ("scan", 360, 360, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("scan", 3200, 3200, 0, 1, 1, True, 0, False, FAST_EMIT_A),
    ("scan", 40000, 40000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("scan", 3200, 3200, 0, 0, 0, False, NT, False, FAST_B),
    ("scan", 3200, 3200, 0, 0, 0, False, 0, True, RING_B),           # duplicate: + the general kernel
    ("scan", 40000, 40000, 0, 0, 1, True, 0, True, FAST_EMIT_B),
    ("scan", 3200, 3200, 0, 1, 1, True, FG, False, None),
    ("ascend_scan", 3200, 3200, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("ascend_scan", 40000, 40000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
]


def _row_id(row):
    entry, stride, n, off, mode_a, ascend, emit, flags, dup, kernel = row
    return (f"{entry}-{stride}x{n}{f'+{off}B' if off else ''}-{'A' if mode_a else 'B'}{'-asc' if ascend else ''}"
            f"{'-emit' if emit else ''}{f'-f{flags}' if flags else ''}{'-dup' if dup else ''}")


@pytest.fixture(scope="module")
def dispatch_ctx(R):
    c = R.Context(0, 70002, 4)
    yield c
    c.close()


# single scans in a context of exactly their size: the stride the rule sees is the count rounded up to even, so the
# shared-memory and cluster kernels serve them as they serve a batch at that stride
SIZED_SINGLE = [
    ("laserscan", 3200, 3200, 0, 0, 0, False, 0, False, SMALL),
    ("laserscan", 8192, 8192, 0, 1, 0, False, 0, False, SMALL),
    ("laserscan", 8191, 8191, 0, 0, 0, False, 0, False, SMALL),      # stride 8192
    ("scan", 3200, 3200, 0, 1, 0, False, 0, False, SMALL),
    ("scan", 8192, 8192, 0, 0, 1, True, 0, False, SMALL),
    ("scan", 3200, 3200, 0, 0, 0, False, NT, False, SMALL),         # NO_TMA does not keep it off the shared memory
    ("scan", 3200, 3200, 0, 0, 1, True, 0, True, SMALL),            # duplicate: + the general kernel
    ("scan", 3200, 3200, 0, 0, 1, True, NS, False, FAST_EMIT_B),
    ("scan", 3200, 3200, 0, 0, 0, False, NS, False, RING_B),
    ("ascend_scan", 3200, 3200, 0, 0, 1, True, 0, False, SMALL),
    ("ascend_scan", 8192, 8192, 0, 0, 1, True, 0, False, SMALL),
    ("laserscan", 20000, 20000, 0, 0, 0, False, 0, False, CLUSTER),
    ("laserscan", 8193, 8193, 0, 0, 0, False, 0, False, CLUSTER),   # stride 8194
    ("laserscan", 20000, 20000, 0, 0, 0, False, 0, True, CLUSTER),  # duplicate: + the general kernel
    ("scan", 32768, 32768, 0, 0, 0, False, 0, False, CLUSTER),
    ("laserscan", 20000, 20000, 0, 1, 0, False, 0, False, RING_A),
    ("scan", 20000, 20000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
    ("laserscan", 20000, 20000, 0, 0, 0, False, NT, False, FAST_B),
    ("ascend_scan", 20000, 20000, 0, 0, 1, True, 0, False, FAST_EMIT_B),
]


@gpu
@pytest.mark.parametrize("row", DISPATCH, ids=[_row_id(r) for r in DISPATCH])
def test_dispatch_table(R, oracle, dispatch_ctx, row):
    check_dispatch(R, oracle, dispatch_ctx, row, DISPATCH.index(row))


@gpu
@pytest.mark.parametrize("row", SIZED_SINGLE, ids=[_row_id(r) for r in SIZED_SINGLE])
def test_dispatch_single_scan_in_a_context_of_its_size(R, oracle, row):
    with R.Context(0, row[2], 1) as ctx:
        check_dispatch(R, oracle, ctx, row, len(DISPATCH) + SIZED_SINGLE.index(row))


def check_dispatch(R, oracle, ctx, row, i):
    """One row of the dispatch table in `ctx`: its results against the oracle and the kernels that ran.  i seeds the
    scan and picks the protocol and the inversion."""
    entry, stride, n, off, mode_a, ascend, emit, flags, dup, kernel = row
    newp, inv = i & 1, (i >> 1) & 1
    scan = tie_free(oracle, n, 60000 + i)
    if dup:
        scan = with_duplicate(scan)
    nodes = np.zeros((2, stride), oracle.NODE_DTYPE)
    nodes[:, :n] = scan
    counts = np.full(2, n, np.uint32)
    single = entry in ("scan", "laserscan", "ascend_scan")
    handed_on = expected_path(kernel, scan, n) == 1
    want = {kernel} - {None}
    if not single or handed_on:
        want.add(GENERAL)
    if single:
        ran = kernels_run(lambda: check_single(R, oracle, ctx, entry, scan, newp, mode_a, inv, ascend, flags), ctx)
    elif entry == "batch":
        ran = kernels_run(lambda: check_batch(R, oracle, ctx, nodes, counts, newp, mode_a, inv, ascend, flags=flags,
                                              emit=emit, expect_path=expected_path(kernel, scan, n)), ctx)
    elif entry == "dev":
        ran = dev_batch(R, oracle, ctx, nodes, counts, [0, 1], newp, mode_a, inv, ascend, flags=flags, emit=emit,
                        offset=off, expect_path=[expected_path(kernel, scan, n)] * 2, profile=True)
    elif entry == "status":
        got = {}
        ran = kernels_run(lambda: got.update(ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts,
                                                            R.scan_params(newp, mode_a, inv, ascend, flags),
                                                            emit_nodes=emit, want_scan=False)), ctx)
        exp = oracle_scans(oracle, nodes, counts, newp, mode_a, inv, ascend)
        assert (got["status"] == exp["status"]).all()
        if emit:  # without ascend the buffer passes through unchanged
            assert (got["nodes"].view(np.uint64) == nodes.view(np.uint64)).all()
    else:
        cp = dict(range_min=0.15, range_max=40.0, intensity_min=10.0, is_new_protocol=newp)
        got = {}
        ran = kernels_run(lambda: got.update(zip(("xyzi", "pc"), ctx.cloud_batch(
            nodes.view(R.NODE_DTYPE), counts, R.cloud_params(flags=R.CLOUD_NO_FUSED if flags & NS else 0, **cp)))), ctx)
        for s in range(2):
            e = oracle.cloud(nodes[s, :n], oracle.cloud_params(**cp))
            assert got["pc"][s] == e.shape[0]
            assert (got["xyzi"][s, : e.shape[0]].view(np.uint32) == e.view(np.uint32)).all()
    assert ran == want, (ran, want)


# ---- C. the 32769..65536-node band, device-resident ----------------------------------------------------------------
def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def band_ctx(R):
    # 3 x (two ring CTAs per SM, the Mode A occupancy) scans: every persistent CTA streams at least three scans
    c = R.Context(0, KEYS, 6 * _sms())
    yield c
    c.close()


def _band_paths(pool, counts, dup, kernel):
    return np.array([1 if d else expected_path(kernel, pool[p], int(counts[p])) for p, d in enumerate(dup)])


@gpu
@pytest.mark.parametrize("stride", BAND_STRIDES)
def test_band_ring_kernel_device_resident(R, oracle, band_ctx, stride):
    """More scans than the ring grid holds (3 x 2 x SMs): each persistent CTA's 16- (Mode B) or 4-stage (Mode A) ring
    wraps inside every large scan and runs ahead across scan boundaries; ragged, odd, empty, unmeasured and duplicate
    cases interleaved in every CTA's sequence."""
    pool, counts, dup = band_pool(oracle, stride, 70000 + stride)
    S = 6 * _sms()
    idx = np.arange(S) % POOL
    for newp, mode_a, inv in ALL_MODES:
        kernel = RING_A if mode_a else RING_B
        paths = _band_paths(pool, counts, dup, kernel)
        for ascend in (0, 1):
            ran = dev_batch(R, oracle, band_ctx, pool, counts, idx, newp, mode_a, inv, ascend, expect_path=paths,
                            profile=(newp, inv, ascend) == (0, 0, 0))
            if ran is not None:
                assert ran == {kernel, GENERAL}, ran
    if stride >= 40000:  # Mode A with M > 32768 really is handed on here, and served below it
        assert (_band_paths(pool, counts, dup, RING_A) == 1).sum() > dup.sum()
        assert (_band_paths(pool, counts, dup, RING_A) == 0).sum() >= 5


@gpu
@pytest.mark.parametrize("stride", BAND_STRIDES)
def test_band_fast_kernel_device_resident(R, oracle, band_ctx, stride):
    """The same cases through scan_fast_kernel: with the ascended buffer (emit), NO_TMA, and a base 8 bytes off a
    16-byte boundary."""
    pool, counts, dup = band_pool(oracle, stride, 80000 + stride)
    S = 3 * _sms()
    idx = (np.arange(S) * 7) % POOL
    for newp, mode_a, inv in ((0, 0, 0), (1, 1, 1), (0, 1, 0), (1, 0, 1)):
        # with the ascended buffer a fill key may land on a measured key: such a scan may go either way
        emit_paths = np.where(dup, 1, -1)
        ran = dev_batch(R, oracle, band_ctx, pool, counts, idx, newp, mode_a, inv, 1, emit=True,
                        expect_path=emit_paths, profile=True)
        assert ran == {FAST_EMIT_A if mode_a else FAST_EMIT_B, GENERAL}, ran
        fast = FAST_A if mode_a else FAST_B
        paths = _band_paths(pool, counts, dup, fast)
        ran = dev_batch(R, oracle, band_ctx, pool, counts, idx, newp, mode_a, inv, 0, flags=NT, expect_path=paths,
                        profile=True)
        assert ran == {fast, GENERAL}, ran
        ran = dev_batch(R, oracle, band_ctx, pool, counts, idx, newp, mode_a, inv, 1, offset=8, expect_path=paths,
                        profile=True)
        assert ran == {fast, GENERAL}, ran


# ---- D. the full key space -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big_ctx(R):
    c = R.Context(0, KEYS + 2, 4)
    yield c
    c.close()


@gpu
def test_full_key_space(R, oracle, big_ctx):
    """65536 measured nodes, every key once: M = 65536, all 2048 bit-words full, inverted Mode B writes from slot
    65535.  Served by the ring kernel (Mode B) and scan_fast_kernel; the ring kernel's Mode A hands it on (M > 32768).
    One duplicated key: handed on everywhere.  65537 nodes with no measured key twice: handed on by the count."""
    ctx = big_ctx
    full = full_key_space(oracle)
    nodes = np.stack([full, with_duplicate(full, 7, 40000)])
    counts = np.full(2, KEYS, np.uint32)
    for newp, inv in ((0, 0), (1, 1), (0, 1), (1, 0)):
        for ascend in (0, 1):
            ran = kernels_run(lambda: check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, emit=False,
                                                  expect_path=[0, 1]), ctx)
            assert ran == {RING_B, GENERAL}, ran
            got = check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, flags=NT, emit=False,
                              expect_path=[0, 1])
            assert got["beam_counts"][0] == KEYS
            check_batch(R, oracle, ctx, nodes, counts, newp, 0, inv, ascend, emit=True, expect_path=[0, 1])
            check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, emit=False, expect_path=[1, 1])
            check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, flags=NT, emit=False, expect_path=[0, 1])
            # (without ascend the buffer passes through and the ring kernel produces the LaserScan: handed on)
            check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, emit=True,
                        expect_path=[0, 1] if ascend else [1, 1])
    # 65537 nodes: the ring kernel (even stride) and scan_fast_kernel (odd stride) must hand it on
    extra = one_node_too_many(oracle)
    for stride in (KEYS + 2, KEYS + 1):
        nodes = np.zeros((1, stride), oracle.NODE_DTYPE)
        nodes[0, : KEYS + 1] = extra
        for newp, mode_a, inv in ALL_MODES:
            check_batch(R, oracle, ctx, nodes, [KEYS + 1], newp, mode_a, inv, 1, emit=False, expect_path=1)
            check_batch(R, oracle, ctx, nodes, [KEYS + 1], newp, mode_a, inv, 1, emit=True, expect_path=1)
    # the ascended buffer with 5 % unmeasured nodes: the fill keys land on measured keys; bit-exact on either path
    sparse = np.roll(oracle.synth_batch(4243, 2, KEYS, 0), -999, axis=1)
    for newp, mode_a, inv in ALL_MODES:
        check_batch(R, oracle, ctx, sparse, np.full(2, KEYS, np.uint32), newp, mode_a, inv, 1, emit=True)


# ---- E. the ring kernel's Mode A index map at its limit ------------------------------------------------------------
# (measured points, key 0 measured): the first two are served, the last two handed on
MODE_A_CASES = [(MODE_A_MAP_MAX, True), (MODE_A_MAP_MAX, False), (MODE_A_MAP_MAX + 1, True), (MODE_A_MAP_MAX + 1, False)]


@gpu
@pytest.mark.parametrize("n", [40000, KEYS])
def test_mode_a_index_map_limit(R, oracle, big_ctx, n):
    """Exactly 32768 measured points stay on scan_tma_kernel<1> (its u16 index map holds one node index per u-rank);
    32769 are handed on.  Measured nodes up to buffer index n - 1, key 0 measured or not (it moves the inverted
    u-ranks), bins of two and three points and a long run of empty bins."""
    ctx = big_ctx
    nodes = np.stack([mode_a_limit_scan(oracle, n, m, k0, 90 + i) for i, (m, k0) in enumerate(MODE_A_CASES)])
    counts = np.full(len(MODE_A_CASES), n, np.uint32)
    for newp, inv in ((0, 0), (1, 1), (0, 1), (1, 0)):
        for ascend in (0, 1):
            ran = kernels_run(lambda: check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, ascend, emit=False,
                                                  expect_path=[0, 0, 1, 1]), ctx)
            assert ran == {RING_A, GENERAL}, ran
        check_batch(R, oracle, ctx, nodes, counts, newp, 1, inv, 0, flags=NT, emit=False, expect_path=0)


# ---- F. the single-scan entry points at real sizes -----------------------------------------------------------------
SINGLE_SIZES = (3200, 8192, 16385, 32768, 40000, KEYS)


@gpu
def test_single_scan_at_real_sizes(R, oracle):
    """ctx.scan (with and without the ascended buffer), ctx.laserscan and ctx.ascend_scan at revolution sizes up to
    the full key space, with and without NO_TMA, in a context much larger than the scan (the result comes back in
    three copies) and in one exactly its size (one copy; an odd size rounds the context's stride up to even).  The
    kernel is the one a batch at the context's stride gets: in the large context the ring kernel (grid of 1) or, with
    NO_TMA or the ascended buffer, scan_fast_kernel; in the exact one up to 8192 nodes the shared-memory kernel, and
    Mode B without the ascended buffer up to 32768 nodes the cluster kernel (grid of 2).  A scan with a duplicated key
    is re-run by the general kernel."""
    scans = {n: [oracle.synth_batch(5100 + n, 1, n, 1)[0]] for n in SINGLE_SIZES}
    for n in SINGLE_SIZES:
        scans[n].append(with_duplicate(measured_everywhere(scans[n][0]), 3, n - 2))
    large = R.Context(0, 4 * KEYS, 1)
    try:
        for n in SINGLE_SIZES:
            exact = R.Context(0, n, 1)
            try:
                for ctx in (large, exact):
                    for k, scan in enumerate(scans[n]):
                        modes = ALL_MODES if k == 0 else [(0, 0, 0), (1, 1, 1), (0, 1, 0), (1, 0, 1)]
                        for flags in (0, NT):
                            for newp, mode_a, inv in modes:
                                check_single(R, oracle, ctx, "scan", scan, newp, mode_a, inv, 0, flags)
                                check_single(R, oracle, ctx, "scan", scan, newp, mode_a, inv, 1, flags)
                                check_single(R, oracle, ctx, "laserscan", scan, newp, mode_a, inv, 0, flags)
                        check_single(R, oracle, ctx, "ascend_scan", scan, 0, 0, 0, 1)
            finally:
                exact.close()
    finally:
        large.close()


# ---- G. PointCloud2 above the shared-memory kernels ----------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [40000, KEYS])
def test_cloud_above_the_shared_memory_kernels(R, oracle, n):
    """scan_tma_kernel<2> and the separate SOR and voxel passes of cloud.cu at 40000 and 65536 nodes (every key once),
    in a context whose per-CTA scratch is sized for 65536 nodes."""
    nodes = room_scans(oracle, 2, n, 31 + n)
    counts = np.array([n, n - 1], np.uint32)
    with R.Context(0, KEYS, 2) as ctx:
        check_cloud(R, oracle, ctx, nodes, counts, range_min=0.15, range_max=40.0, intensity_min=10.0)
        ran = kernels_run(lambda: check_cloud(R, oracle, ctx, nodes, counts, range_min=0.15, range_max=40.0,
                                              sor_k=8, sor_alpha=1.0, voxel_size=0.05), ctx)
        assert ran == {RING_CLOUD, GENERAL, SOR, VOXEL}, ran
        check_cloud(R, oracle, ctx, nodes, counts, range_min=0.15, range_max=40.0, sor_k=8, sor_alpha=1.0)
        check_cloud(R, oracle, ctx, nodes, counts, range_min=0.15, range_max=40.0, voxel_size=6.0)


@gpu
def test_cloud_projection_of_every_key_within_1e6_of_float64(R, oracle):
    """Every key once, ranges from 1/4 mm upward, through the CUDA path against float64 numpy directly."""
    from test_cloud_semantics import check_projection

    keys = np.arange(KEYS)
    rng = np.random.default_rng(5)
    dist = np.concatenate([[1, 2, 3, 599, 600, 160000, 160001, 2**31], rng.integers(1, 200000, KEYS - 8)])
    nodes = oracle.make_nodes(keys, dist, rng.integers(0, 256, KEYS), 2)
    nodes = np.roll(nodes, -20000)[None]
    with R.Context(0, KEYS, 1) as ctx:
        for kw in (dict(range_min=0.0, range_max=1e9), dict(range_min=0.15, range_max=40.0, intensity_min=17.0)):
            xyzi, pc = ctx.cloud_batch(nodes.view(R.NODE_DTYPE), np.array([KEYS], np.uint32), R.cloud_params(**kw))
            assert check_projection(xyzi[0, : pc[0]], nodes[0], **kw) < 1e-6


# ---- H. the case builders, without a GPU ---------------------------------------------------------------------------
def test_case_builders_make_what_the_gpu_tests_rely_on(oracle):
    for n in (40000, KEYS):
        for i, (m, with0) in enumerate(MODE_A_CASES):
            s = mode_a_limit_scan(oracle, n, m, with0, 90 + i)
            k = measured_keys(s)
            assert len(s) == n and len(k) == m and len(np.unique(k)) == m
            assert (0 in k) == with0
            pos = np.flatnonzero(s["dist_mm_q2"] != 0)
            assert pos[-1] == n - 1 and (pos >= 32768).sum() > 1000
            present = np.zeros(KEYS, bool)
            present[k] = True
            assert present[int(not with0): int(not with0) + 20000].all() and not present[40000:52000].any()
    full = full_key_space(oracle)
    assert (np.sort(full["angle_z_q14"]) == np.arange(KEYS)).all() and (full["dist_mm_q2"] != 0).all()
    assert not has_duplicate(full) and has_duplicate(with_duplicate(full, 7, 40000))
    extra = one_node_too_many(oracle)
    assert len(extra) == KEYS + 1 and len(measured_keys(extra)) == KEYS and not has_duplicate(extra)
    for stride in BAND_STRIDES:
        pool, counts, dup = band_pool(oracle, stride, 70000 + stride)
        assert pool.shape == (POOL, stride) and (counts <= stride).all()
        assert set(counts.tolist()) >= {min(c, stride) for c in BAND_COUNTS} | {stride}
        assert (counts % 2 == 1).sum() >= 5
        assert dup.sum() == 1
        for p in range(POOL):
            assert has_duplicate(pool[p], counts[p]) == dup[p], (stride, p)
            assert (pool[p]["dist_mm_q2"][counts[p]:] != 0).all()  # measured nodes behind the count
        d = np.flatnonzero(dup)[0]
        twin = np.flatnonzero(pool[d]["angle_z_q14"] == pool[d]["angle_z_q14"][5])
        assert len(twin) == 2 and twin[0] == 5 and twin[1] // CH == min(40, (stride - 1) // CH)
        assert (pool[d]["dist_mm_q2"][twin] != 0).all()
        nothing = [p for p in range(POOL) if counts[p] == stride and not measured_keys(pool[p], counts[p]).size]
        tail = [p for p in range(POOL) if counts[p] == stride and (pool[p]["dist_mm_q2"][-3 * CH:] == 0).all()]
        assert len(nothing) == 1 and len(set(tail) - set(nothing)) == 1
    for i, row in enumerate(DISPATCH + SIZED_SINGLE):
        entry, stride, n, off, mode_a, ascend, emit, flags, dup, kernel = row
        assert n <= stride and (entry == "dev" or off == 0)
        assert i < len(DISPATCH) or (entry in ("scan", "laserscan", "ascend_scan") and n == stride)
        scan = tie_free(oracle, n, 60000 + i)
        assert has_duplicate(scan) == (n > KEYS)
