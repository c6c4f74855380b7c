"""The scan kernels over the whole arithmetic domain of their shortcuts, bit for bit against the reference's float chain.

Mode A: every beam count M the shared-memory kernel serves (1..8192) and a dense selection up to 65536 for the ring
kernel scan_tma_kernel<1>, scan_fast_kernel, its emit variant (the ascended buffer) and the general kernel, both
orientations; for each (M, orientation) the cover scans of tests/test_domain_sweep_pieces.py put every one of the
65536 keys into its bin, so every key meets every bin edge the integer quotient of mode_a_bin_fast could get wrong.
Tie scans (two keys of one bin on one distance) check the lower key's win on the shared-memory and the ring kernel.

Mode B: every distinct nonzero float32 a u32 distance converts to (the 2^24 integers from 1, then every float up to
2^32, reached by 2^32 - 1), through dist_to_m of the shared-memory, the ring and the general kernel, upright and
inverted, all 256 qualities under both protocols; and the Mode B angle_increment of the swept beam counts above 8192.

The scans are built on the device with torch; the expectations come from numpy.  The first launch of every sweep runs
once more under the CUDA profiler, in a child process, to confirm the kernel family it is meant to reach; every launch
is checked for `path` of every scan.  Each prints
its runtime, its case count and the device memory it held (-s shows them)."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from test_domain_sweep_pieces import (KEYS, MODE_A_MAP_MAX, RING_MS, SMALL_MS, WIDE_MS, Cover, F32, Tables, cover_scans,
                                      describe_mode_a_mismatch, first_mode_a_mismatch, mode_a_increment,
                                      mode_b_increment, node_dist, node_quality, pack_nodes, rolled, tie_scan)
from test_gpu_scan_bands import CLUSTER, FAST_A, FAST_EMIT_A, GENERAL, RING_A, RING_B, SMALL, kernels_run

gpu = pytest.mark.gpu

NS, NT, FG = 4, 2, 1   # RPL_FLAG_NO_SMALL, RPL_FLAG_NO_TMA, RPL_FLAG_FORCE_GENERAL
SLOTS = 4 << 20        # node slots per launch: ~0.3 GB of buffers and temporaries at the peak of a check
MAX_SCANS = 1 << 17    # M = 1 takes 65536 cover scans


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


class Meter:
    """Wall time, and the device memory a sweep holds at its peak: what the library's context took (its allocations
    do not go through torch's allocator, so the free memory the driver reports is sampled around its creation) plus
    the most torch held for the sweep's buffers at once."""

    def __init__(self):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()
        self.base = torch.cuda.memory_allocated()
        self.ctx_bytes = 0

    def context(self, R, *args):
        free0 = torch.cuda.mem_get_info()[0]
        ctx = R.Context(0, *args)
        self.ctx_bytes = free0 - torch.cuda.mem_get_info()[0]
        return ctx

    def report(self, what, cases):
        held = torch.cuda.max_memory_allocated() - self.base
        torch.cuda.empty_cache()
        print(f"\n[domain sweep] {what}: {cases} cases, {time.perf_counter() - self.t0:.1f} s, device memory: "
              f"context {self.ctx_bytes / 2**20:.0f} MiB + buffers {held / 2**20:.0f} MiB, on "
              f"{torch.cuda.get_device_name()}")


def profiled(fn, ctx, want):
    """The kernels that ran in fn(), under the CUDA profiler.  The profiler now and then drops a kernel's activity
    record (a capture then holds a strict subset of the kernels the library launched, sometimes none of them): such a
    capture says nothing, and the call is profiled again, up to three times.  A capture with any kernel outside
    `want` is returned at once."""
    for _ in range(3):
        ran = kernels_run(fn, ctx)
        if not ran < want:
            break
    return ran


def kernels_in_a_child_process():
    """{case: kernels that ran} for the first launch of every sweep, each profiled in a Python process of its own.
    The sweeps run minutes of heavy device work; profiling them in the test process left CUDA activity tracing
    recording no kernels for the profiler tests of other files later in the same process.  A child process takes
    its tracing state with it when it exits."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"),
                                                       os.environ.get("PYTHONPATH", "")]))
    code = ("import json, test_gpu_domain_sweeps as T; "
            "print('KERNELS ' + json.dumps(T.first_launch_kernels()), flush=True)")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, env=env, capture_output=True, text=True,
                       timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")]
    assert r.returncode == 0 and lines, f"the profiling process failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return {k: set(v) for k, v in json.loads(lines[-1][len("KERNELS "):]).items()}


@pytest.fixture(scope="module")
def kernels_seen():
    return kernels_in_a_child_process()


def bits_of(values):
    return torch.from_numpy(np.asarray(values, F32).view(np.int32).astype(np.int64))


def launch(R, ctx, nodes, counts, stride, params, emit):
    """scan_batch_dev over device buffers; returns (ranges, intensities, beams, inc, status, path, nodes_out)."""
    dev = nodes.device
    S = nodes.shape[0]
    ranges = torch.full((S, stride), float("nan"), dtype=torch.float32, device=dev)
    intens = torch.full((S, stride), float("nan"), dtype=torch.float32, device=dev)
    beams, status, path = (torch.full((S,), -1, dtype=torch.int32, device=dev) for _ in range(3))
    inc = torch.full((S,), float("nan"), dtype=torch.float32, device=dev)
    nodes_out = torch.zeros_like(nodes) if emit else None
    torch.cuda.synchronize()  # the buffers were filled on torch's stream; the library runs on its own
    ctx.scan_batch_dev(nodes.data_ptr(), counts.data_ptr(), S, stride, params,
                       nodes_out=None if nodes_out is None else nodes_out.data_ptr(), ranges=ranges.data_ptr(),
                       intensities=intens.data_ptr(), beam_counts=beams.data_ptr(), angle_increment=inc.data_ptr(),
                       status=status.data_ptr(), path=path.data_ptr())
    ctx.synchronize()
    torch.cuda.synchronize()
    return ranges, intens, beams, inc, status, path, nodes_out


# ---- Mode A ------------------------------------------------------------------------------------------------------------
# name: (beam counts, the kernel that must serve every scan (None: the general kernel alone), flags and stride of the
# g-th launch group from its largest M, ascended buffer, tie scans)
FAMILIES = {
    "shared-memory": (SMALL_MS, SMALL, lambda g, m: (0, m), False, True),
    "ring": (RING_MS, RING_A, lambda g, m: (NS, m + (m & 1)), False, True),
    # odd strides leave every second scan 8 bytes off a 16-byte boundary; even ones take NO_TMA (as does M = 65536:
    # a context for 65537 nodes would take another 1.3 GiB of scratch)
    "fast": (WIDE_MS, FAST_A, lambda g, m: (NS, m | 1) if g % 2 == 0 and m < KEYS else (NS | NT, m + (m & 1)), False,
             False),
    "emit": (WIDE_MS, FAST_EMIT_A, lambda g, m: (NS, m + (m & 1)), True, False),
    "general": (WIDE_MS, None, lambda g, m: (FG, m), False, False),
}


def groups(ms, inverted, ties):
    """Consecutive beam counts that share one launch: the largest within 1.25 x the smallest, at most SLOTS node
    slots and MAX_SCANS scans.  Yields lists of Covers."""
    group, rows, m0 = [], 0, 0
    for m in ms:
        cov = Cover(m, inverted)
        w = cov.n_scans + (1 if ties and m <= MODE_A_MAP_MAX else 0)
        if group and (m > m0 * 5 // 4 + 2 or (rows + w) * m > SLOTS or rows + w > MAX_SCANS):
            yield group
            group, rows = [], 0
        if not group:
            m0 = m
        group.append(cov)
        rows += w
    if group:
        yield group


def build_group(covers, stride, ties, dev):
    """(nodes [S, stride] int64 words, counts [S] int32, winner [S, stride], ms [S]) of the covers' scans and, with
    ties, one tie scan per M <= 32768.  Every node is measured; the slots behind a scan's count stay zero."""
    parts = []
    for cov in covers:
        keys, win = cover_scans(cov, dev)
        parts.append((keys, node_dist(keys), node_quality(keys), win))
        if ties and cov.m <= MODE_A_MAP_MAX:
            parts.append(tie_scan(cov, dev))
    S = sum(p[0].shape[0] for p in parts)
    nodes = torch.zeros((S, stride), dtype=torch.int64, device=dev)
    winner = torch.full((S, stride), -1, dtype=torch.int64, device=dev)
    ms = torch.empty(S, dtype=torch.int64, device=dev)
    r0 = 0
    for keys, dist, qual, win in parts:
        W, M = keys.shape
        seed = M * 31 + r0
        nodes[r0:r0 + W, :M] = pack_nodes(rolled(keys, seed), rolled(dist, seed), rolled(qual, seed))
        winner[r0:r0 + W, :M] = win
        ms[r0:r0 + W] = M
        r0 += W
    return nodes, ms.to(torch.int32), winner, ms


def sorted_nodes(nodes, ms):
    """The ascended buffer of scans whose nodes are all measured on distinct keys: the nodes by ascending key."""
    col = torch.arange(nodes.shape[1], device=nodes.device)[None, :]
    k = torch.where(col < ms[:, None], nodes & 0xFFFF, torch.full_like(nodes, KEYS + 1))
    return nodes.gather(1, k.argsort(1))


def check_scan_outputs(out, ms, winner, newp, inverted, want_path, inc_bits, tab, what):
    ranges, intens, beams, inc, status, path, _ = out
    assert bool((status == 0).all()), (what, "status")
    bad = (beams.to(torch.int64) != ms).nonzero()
    assert bad.numel() == 0, f"{what}: M={int(ms[bad[0]])}: beam_count {int(beams[bad[0]])}"
    bad = (inc.view(torch.int32).to(torch.int64) != inc_bits).nonzero()
    assert bad.numel() == 0, f"{what}: M={int(ms[bad[0]])}: angle_increment {float(inc[bad[0]])!r}"
    bad = (path != want_path).nonzero()
    assert bad.numel() == 0, f"{what}: M={int(ms[bad[0]])}: path {int(path[bad[0]])}, want {want_path}"
    where = first_mode_a_mismatch(ranges, intens, winner, ms, newp, tab)
    if where is not None:
        pytest.fail(describe_mode_a_mismatch(where, ranges, winner, ms, inverted, what, tab))


def mode_a_group(R, family, inverted, g, covers, dev):
    """(nodes, counts, winner, ms, stride, params, newp) of launch group g of a Mode A sweep."""
    _, _, flags_of, emit, ties = FAMILIES[family]
    newp = g & 1
    flags, stride = flags_of(g, covers[-1].m)
    nodes, counts, winner, ms = build_group(covers, stride, ties, dev)
    params = R.scan_params(newp, 1, int(inverted), 1 if emit else (g >> 1) & 1, flags)
    return nodes, counts, winner, ms, stride, params, newp


@gpu
@pytest.mark.parametrize("inverted", [False, True], ids=["upright", "inverted"])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_mode_a_every_key_at_every_bin_edge(R, kernels_seen, family, inverted):
    """Every key of every swept M lands in the bin the float chain gives it, through the kernel family's own
    binning (mode_a_bin_fast and the scatter-min / index map / emit logic around it; the general kernel's plain
    float chain); ties go to the lower key."""
    ms_list, kernel, flags_of, emit, ties = FAMILIES[family]
    assert kernels_seen[f"A {family} {int(inverted)}"] == {kernel, GENERAL} - {None}, kernels_seen
    dev = torch.device("cuda")
    tab = Tables(dev)
    meter = Meter()
    max_stride = max(flags_of(g, max(ms_list))[1] for g in (0, 1))
    cases = 0
    with meter.context(R, max_stride, MAX_SCANS) as ctx:
        for g, covers in enumerate(groups(ms_list, inverted, ties)):
            nodes, counts, winner, ms, stride, params, newp = mode_a_group(R, family, inverted, g, covers, dev)
            what = f"{kernel or GENERAL} (Mode A, stride {stride}, flags {params.flags}, protocol {'new' if newp else 'old'})"
            out = launch(R, ctx, nodes, counts, stride, params, emit)
            inc_bits = bits_of([mode_a_increment(c.m) for c in covers]).to(dev)
            per_m = torch.bincount(ms, minlength=covers[-1].m + 1)[[c.m for c in covers]]
            check_scan_outputs(out, ms, winner, newp, inverted, 1 if kernel is None else 0,
                               torch.repeat_interleave(inc_bits, per_m), tab, what)
            if emit:
                live = torch.arange(stride, device=dev)[None, :] < ms[:, None]
                ok = torch.where(live, out[6] == sorted_nodes(nodes, ms), torch.ones_like(live))
                assert bool(ok.all()), f"{what}: ascended buffer of M={int(ms[(~ok).any(1).nonzero()[0]])}"
            cases += KEYS * len(covers)
            del nodes, winner, out
    meter.report(f"Mode A {family} {'inverted' if inverted else 'upright'} ({len(ms_list)} beam counts)",
                 f"{cases} (M, key)")


MODE_B_MS = [m for m in WIDE_MS if m > 8192]


@gpu
def test_mode_b_angle_increment_above_the_shared_memory_kernel(R, kernels_seen):
    """Mode B of the cover scans of the swept beam counts above 8192 (the cluster and the ring kernel): the
    angle_increment 2*pi / (M - 1), and every node in key order (reversed when inverted)."""
    # LaserScan Mode B at strides up to 32768 takes the two-CTA cluster kernel, larger ones the ring
    assert kernels_seen["B increment"] == {CLUSTER, GENERAL}, kernels_seen
    dev = torch.device("cuda")
    tab = Tables(dev)
    meter = Meter()
    n = 0
    with meter.context(R, KEYS, MAX_SCANS) as ctx:
        for inverted in (False, True):
            for g, covers in enumerate(groups(MODE_B_MS, inverted, False)):
                stride = covers[-1].m + (covers[-1].m & 1)
                nodes, counts, _, ms = build_group(covers, stride, False, dev)
                newp = g & 1
                params = R.scan_params(newp, 0, int(inverted), 0, 0)
                out = launch(R, ctx, nodes, counts, stride, params, False)
                keys = sorted_nodes(nodes, ms) & 0xFFFF
                col = torch.arange(stride, device=dev)[None, :]
                if inverted:
                    keys = keys.gather(1, torch.where(col < ms[:, None], ms[:, None] - 1 - col, col))
                slot_key = torch.where(col < ms[:, None], keys, torch.full_like(keys, -1))
                inc_bits = torch.repeat_interleave(bits_of([mode_b_increment(c.m) for c in covers]).to(dev),
                                                   torch.tensor([c.n_scans for c in covers], device=dev))
                check_scan_outputs(out, ms, slot_key, newp, inverted, 0, inc_bits, tab,
                                   f"Mode B stride {stride} {'inverted' if inverted else 'upright'}")
                n += len(covers)
    meter.report("Mode B angle_increment above 8192", f"{n} (M, orientation)")


# ---- Mode B: every distance --------------------------------------------------------------------------------------------
def every_distance():
    """One u32 for every distinct nonzero float32 a u32 converts to, ascending: 1..2^24, every float in (2^24, 2^32)
    (all integers), and 2^32 - 1 for 2^32.  83,886,080 values = 1280 x 65536."""
    lo = np.arange(1, (1 << 24) + 1, dtype=np.uint32)
    hi = np.arange(0x4B800001, 0x4F800000, dtype=np.uint32).view(np.float32).astype(np.uint32)
    return np.concatenate([lo, hi, np.array([0xFFFFFFFF], np.uint32)])


@pytest.fixture(scope="module")
def distances():
    d = every_distance()
    assert len(d) == 83886080 and (np.diff(d.astype(np.int64)) > 0).all()
    assert len(np.unique(d.astype(np.float32))) == len(d)
    return d, (d.astype(F32) / F32(4000.0)).view(np.int32)


# name: (kernel, nodes per scan = stride, flags)
MODE_B_KERNELS = {"shared-memory": (SMALL, 8192, 0), "ring": (RING_B, KEYS, 0), "general": (None, KEYS, FG)}
COMBOS = [(0, False), (1, True), (1, False), (0, True)]  # (new protocol, inverted) of successive launches


def mode_b_chunk(d_host, K, j0, C, ci, dev):
    """(nodes, dist, qual) of scans j0..j0 + C of the distance sweep, dist and qual [C, K] by key rank."""
    rank = torch.arange(K, device=dev)
    j = torch.arange(j0, j0 + C, device=dev)[:, None]
    dist = torch.from_numpy(d_host[j0 * K:(j0 + C) * K].astype(np.int64)).to(dev).view(C, K)
    keys = rank[None, :] * (KEYS // K) + j % (KEYS // K)   # ascending in the rank
    qual = (rank[None, :] + j) & 0xFF
    seed = 7 * ci + 1
    return pack_nodes(rolled(keys, seed), rolled(dist, seed), rolled(qual, seed)), dist, qual


@gpu
@pytest.mark.parametrize("family", list(MODE_B_KERNELS))
def test_mode_b_every_distance(R, distances, kernels_seen, family):
    """Every distinct distance through dist_to_m (a multiply and two FMAs): scan j of K nodes holds K distinct keys
    (every key, or every 8th from j mod 8) at a rotated start, the distance of rank r being value j * K + r and the
    quality (r + j) mod 256; the ranges come back in key order, float32(dist) / 4000 bit for bit."""
    kernel, K, flags = MODE_B_KERNELS[family]
    assert kernels_seen[f"B {family}"] == {kernel, GENERAL} - {None}, kernels_seen
    d_host, e_host = distances
    dev = torch.device("cuda")
    meter = Meter()
    n_scans = len(d_host) // K
    chunk = SLOTS // K
    done = 0
    with meter.context(R, K, chunk) as ctx:
        for ci, j0 in enumerate(range(0, n_scans, chunk)):
            newp, inverted = COMBOS[ci % 4]
            C = min(chunk, n_scans - j0)
            nodes, dist, qual = mode_b_chunk(d_host, K, j0, C, ci, dev)
            counts = torch.full((C,), K, dtype=torch.int32, device=dev)
            params = R.scan_params(newp, 0, int(inverted), ci & 1, flags)
            out = launch(R, ctx, nodes, counts, K, params, False)
            ranges, intens, beams, inc, status, path, _ = out
            what = f"{kernel or GENERAL} (Mode B, {'inverted' if inverted else 'upright'}, protocol {'new' if newp else 'old'})"
            assert bool((status == 0).all()) and bool((beams == K).all()), what
            assert bool((inc.view(torch.int32) == int(np.asarray(mode_b_increment(K)).view(np.int32))).all()), what
            assert bool((path == (1 if kernel is None else 0)).all()), what
            exp_r = torch.from_numpy(e_host[j0 * K:(j0 + C) * K]).to(dev).view(C, K)
            exp_i = (qual if newp else qual >> 2).to(torch.float32).view(torch.int32)
            if inverted:
                exp_r, exp_i = exp_r.flip(1), exp_i.flip(1)
            ok = (ranges.view(torch.int32) == exp_r) & (intens.view(torch.int32) == exp_i)
            if not bool(ok.all()):
                s, slot = (int(v) for v in (~ok).nonzero()[0])
                r = K - 1 - slot if inverted else slot
                pytest.fail(f"{what}: scan {j0 + s} slot {slot}: dist_mm_q2 {int(dist[s, r])} quality {int(qual[s, r])}"
                            f" -> range bits {int(ranges[s, slot].view(torch.int32)):#010x}, intensity "
                            f"{float(intens[s, slot])}; want {int(exp_r[s, slot]):#010x}, {float(exp_i[s, slot].view(torch.float32))}")
            done += C * K
            del nodes, dist, out, exp_r, exp_i
    assert done == len(d_host)
    meter.report(f"Mode B {family} every distance", f"{done} distances")


def first_launch_kernels():
    """{case: sorted kernels that ran} for the first launch group of every sweep above, each under the CUDA profiler
    (run by kernels_in_a_child_process)."""
    import rplidar_ros2_driver_b200 as R

    dev = torch.device("cuda")
    seen = {}
    for family, (ms_list, kernel, _, emit, ties) in FAMILIES.items():
        for inverted in (False, True):
            covers = next(groups(ms_list, inverted, ties))
            nodes, counts, _, _, stride, params, _ = mode_a_group(R, family, inverted, 0, covers, dev)
            with R.Context(0, stride, nodes.shape[0]) as ctx:
                want = {kernel, GENERAL} - {None}
                seen[f"A {family} {int(inverted)}"] = profiled(
                    lambda: launch(R, ctx, nodes, counts, stride, params, emit), ctx, want)
    covers = next(groups(MODE_B_MS, False, False))
    stride = covers[-1].m + (covers[-1].m & 1)
    nodes, counts, _, _ = build_group(covers, stride, False, dev)
    with R.Context(0, stride, nodes.shape[0]) as ctx:
        seen["B increment"] = profiled(lambda: launch(R, ctx, nodes, counts, stride, R.scan_params(0, 0, 0, 0, 0), False),
                                       ctx, {CLUSTER, GENERAL})
    d = np.arange(1, 2 * KEYS + 1, dtype=np.uint32)
    for family, (kernel, K, flags) in MODE_B_KERNELS.items():
        C = len(d) // K
        nodes, _, _ = mode_b_chunk(d, K, 0, C, 0, dev)
        counts = torch.full((C,), K, dtype=torch.int32, device=dev)
        with R.Context(0, K, C) as ctx:
            seen[f"B {family}"] = profiled(lambda: launch(R, ctx, nodes, counts, K, R.scan_params(0, 0, 0, 0, flags), False),
                                           ctx, {kernel, GENERAL} - {None})
    return {k: sorted(v) for k, v in seen.items()}
