"""The PointCloud2 chain at the limits of the fused shared-memory kernel (scan_small.cu, POST), with the kernels that
ran made visible.

Every case is compared bit for bit with oracle/cloud_oracle.cpp on both implementations (check_cloud: the fused chain
and CLOUD_NO_FUSED = scan kernel + separate passes) AND checked by the float64 checkers of tests/test_cloud_checkers.py,
which share nothing with the oracle.  The cases:

  * one voxel cell of 4096 members with an intensity sum of 1,044,480 (the fused kernel packs members and intensity
    sum as (members - 1) << 20 | sum in 32 bits);
  * per-leader 16.16 fixed-point delta sums past 1.0e9 in every quadrant (its int accumulators wrap at 2^31);
  * points whose float32 x / voxel is an integer or 1-3 ulps either side of one, both signs, four voxel sizes, and the
    near-zero coordinates at 0 / 90 / 180 / 270 degrees (floor_div's guess and its fallback to the division);
  * the host's admission rule (rpl_capi.cu launch_fast: voxel <= 4 m and range_max / voxel < 32000) on both sides of
    both limits: identical results, different kernels;
  * SOR at every k band (sor_k 1, 4, 5, 8, 9, 16, 17, 32: the fused kernel's win8 / generic split and the separate
    pass's K = 4 / 8 / 16 / 32), scans with exactly 2, 3, 32-35 points around the all-others / window switch, and
    isolated spikes (sor_mean_win8 merges a later group only when a lane of the warp needs it);
  * strides 8192 and 32768, which take the plain shared-memory kernel or the ring kernel and the separate passes.

Which kernels ran: the SOR and voxel passes are launched whenever they are asked for -- after the fused kernel they
serve only the scans it handed to the general kernel (duplicate keys) -- so what tells a fused chain from separate
passes is the variant of scan_small_kernel that ran (SMALL_POST = scan_small_kernel<2, false, true, ...>).  The kernel
sets are taken under the CUDA profiler in a child process, once for every case (kernel_sets): profiling here, early in
a pytest process, made the profiler lose kernels that tests/test_gpu_scan_bands.py launches later in it."""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

from test_cloud_checkers import (BOUNDARY_VOXELS, SOR_WINDOW_COUNTS, boundary_scan, check_sor, check_voxel_grid,
                                 corner_scan, packing_limit_scan, spike_scan, trig_table, window_scan)
from test_cloud_semantics import check_projection
from test_gpu_cloud import check_cloud, room_scans
from test_gpu_scan_bands import _B, GENERAL, RING_CLOUD, SMALL, SOR, VOXEL, _short_name

gpu = pytest.mark.gpu

SMALL_POST = "scan_small_kernel<post>"
_SMALL_CLOUD = (re.compile(r"scan_small_kernel\s*<\s*(?:\(int\)\s*)?2\s*,\s*" + _B + r"\s*,\s*" + _B),
                re.compile(r"scan_small_kernelILi2ELb([01])ELb([01])E"))
TESTS = os.path.dirname(os.path.abspath(__file__))
SOR_KS = (1, 4, 5, 8, 9, 16, 17, 32)
CTX_ARGS = (0, 40000, 16)  # device, max_nodes, max_scans


# ---- the cases ------------------------------------------------------------------------------------------------------
def stack(scans, stride=None):
    stride = stride or max(len(s) for s in scans)
    nodes = np.zeros((len(scans), stride), scans[0].dtype)
    for i, s in enumerate(scans):
        nodes[i, : len(s)] = s
    return nodes, np.array([len(s) for s in scans], np.uint32)


def small_room(O, seed):
    """Room scans with every range below 3.9 m: no coordinate within a 4 m voxel's reach of a cell boundary but 0."""
    nodes = room_scans(O, 3, 3200, seed)
    nodes["dist_mm_q2"] = np.minimum(nodes["dist_mm_q2"], 15600)
    return nodes, np.full(3, 3200, np.uint32)


def limit_cases(O):
    """name -> (nodes, counts, kernel the scans start on, cloud parameters)."""
    cases = {}
    cases["packing"] = (*stack([packing_limit_scan(O, 5), packing_limit_scan(O, 6)]), SMALL_POST,
                        dict(range_min=0.0, range_max=40.0, is_new_protocol=1, voxel_size=4.0))
    cases["corners"] = (*stack([corner_scan(O, q) for q in range(4)]), SMALL_POST,
                        dict(range_min=0.0, range_max=40.0, voxel_size=4.0))
    trig = trig_table(O)
    for v in BOUNDARY_VOXELS:
        cases[f"boundary-{v:.4f}"] = (*stack([boundary_scan(O, trig, v, seed=s) for s in (0, 1)]), SMALL_POST,
                                      dict(range_min=0.0, range_max=40.0, voxel_size=v))
    room4 = small_room(O, 61)
    above4 = float(np.nextafter(np.float32(4.0), np.float32(np.inf)))
    sor8 = dict(range_min=0.15, range_max=40.0, sor_k=8, sor_alpha=1.0)
    cases["voxel-4"] = (*room4, SMALL_POST, dict(sor8, voxel_size=4.0))
    cases["voxel-above-4"] = (*room4, SMALL, dict(sor8, voxel_size=above4))
    room32k = small_room(O, 62)
    below = float(np.nextafter(np.float32(31.25), np.float32(0.0)))
    cases["cells-below-32000"] = (*room32k, SMALL_POST, dict(range_min=0.15, range_max=below, voxel_size=2.0 ** -10))
    cases["cells-32000"] = (*room32k, SMALL, dict(range_min=0.15, range_max=31.25, voxel_size=2.0 ** -10))
    scans = [window_scan(O, m, 40 + m) for m in SOR_WINDOW_COUNTS]
    scans += [spike_scan(O, 3200, 7), spike_scan(O, 2900, 8), room_scans(O, 1, 3200, 9)[0]]
    sor_nodes, sor_counts = stack(scans)
    for k in SOR_KS:
        for alpha in (0.0, 1.0, 2.5):
            cases[f"sor-{k}-{alpha}"] = (sor_nodes, sor_counts, SMALL_POST,
                                         dict(range_min=0.15, range_max=40.0, sor_k=k, sor_alpha=alpha))
        cases[f"sor-{k}-voxel"] = (sor_nodes, sor_counts, SMALL_POST,
                                   dict(range_min=0.15, range_max=40.0, sor_k=k, sor_alpha=1.0, voxel_size=0.05))
    for stride, head in ((8192, SMALL), (32768, RING_CLOUD)):
        nodes = room_scans(O, 2, stride, 70 + stride)
        counts = np.array([stride, stride - 1], np.uint32)
        for k, alpha, v in ((8, 1.0, 0.05), (16, 2.5, 0.25), (4, 0.0, 1.0 / 3.0)):
            cases[f"stride-{stride}-{k}"] = (nodes, counts, head, dict(range_min=0.15, range_max=40.0, sor_k=k,
                                                                       sor_alpha=alpha, voxel_size=v))
    return cases


# ---- which kernels ran ----------------------------------------------------------------------------------------------
def _chain_name(name):
    if "scan_small_kernel" in name:
        for rx in _SMALL_CLOUD:
            m = rx.search(name)
            if m:
                return SMALL_POST if m[2] in ("true", "1") else SMALL
        raise AssertionError(f"not a PointCloud2 variant of scan_small_kernel: {name!r}")
    return _short_name(name)


def chain_kernels(fn, ctx) -> set:
    """tests/test_gpu_scan_bands.py::kernels_run, with the fused variant of the shared-memory kernel told apart."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx.synchronize()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.02)  # keep the kernels clear of both edges of the capture window (see kernels_run)
        fn()
        ctx.synchronize()
        torch.cuda.synchronize()
        time.sleep(0.02)
    names = [e.name for e in prof.events()]
    raw = getattr(getattr(prof, "profiler", None), "kineto_results", None)
    if raw is not None:
        names += [e.name() for e in raw.events()]
    return {s for s in map(_chain_name, names) if s}


def child_kernel_sets():
    """(run in a child process) the kernels every case runs, by name."""
    import rplidar_ros2_driver_b200 as R
    from oracle import pyoracle as O

    out = {}
    with R.Context(*CTX_ARGS) as ctx:
        for name, (nodes, counts, _, kw) in limit_cases(O).items():
            out[name] = sorted(chain_kernels(
                lambda: ctx.cloud_batch(nodes.view(R.NODE_DTYPE), counts, R.cloud_params(**kw)), ctx))
    return out


# ---- fixtures -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(*CTX_ARGS)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cases(oracle):
    return limit_cases(oracle)


@pytest.fixture(scope="module")
def kernel_sets(oracle):
    code = (f"import json, sys; sys.path[:0] = [{os.path.dirname(TESTS)!r}, {TESTS!r}]; "
            "import test_gpu_cloud_limits as T; print('KERNEL_SETS ' + json.dumps(T.child_kernel_sets()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600,
                         cwd=os.path.dirname(TESTS))
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("KERNEL_SETS ")]
    assert out.returncode == 0 and line, out.stdout[-3000:] + out.stderr[-3000:]
    return {k: set(v) for k, v in json.loads(line[0][len("KERNEL_SETS "):]).items()}


def run_case(R, O, ctx, cases, kernel_sets, name):
    """Oracle bit for bit on both implementations, the kernel set of the default one, and the float64 checkers on the
    CUDA outputs: projection -> (SOR) -> (voxel grid), each step checked from the CUDA path's own previous step."""
    nodes, counts, head, kw = cases[name]
    check_cloud(R, O, ctx, nodes, counts, **kw)
    sor, voxel = kw.get("sor_k", 0), kw.get("voxel_size", 0.0)
    want = {head, GENERAL} | ({SOR} if sor else set()) | ({VOXEL} if voxel else set())
    assert kernel_sets[name] == want, (name, kernel_sets[name], want)

    def cuda(**over):
        return ctx.cloud_batch(nodes.view(R.NODE_DTYPE), counts, R.cloud_params(**dict(kw, **over)))

    base, bpc = cuda(sor_k=0, voxel_size=0.0)
    mid, mpc = cuda(voxel_size=0.0) if sor else (base, bpc)
    fin, fpc = cuda() if voxel else (mid, mpc)
    window = dict(range_min=kw["range_min"], range_max=kw["range_max"], intensity_min=kw.get("intensity_min", 0.0),
                  new_protocol=kw.get("is_new_protocol", 0))
    for s in range(nodes.shape[0]):
        b = base[s, : bpc[s]]
        check_projection(b, nodes[s, : counts[s]], **window)
        if sor:
            check_sor(b, mid[s, : mpc[s]], sor, kw.get("sor_alpha", 1.0))
        if voxel:
            check_voxel_grid(mid[s, : mpc[s]], fin[s, : fpc[s]], voxel)
    return fin, fpc


# ---- the tests ------------------------------------------------------------------------------------------------------
@gpu
def test_one_cell_at_the_packing_limit(R, oracle, ctx, cases, kernel_sets):
    fin, fpc = run_case(R, oracle, ctx, cases, kernel_sets, "packing")
    assert (fpc == 1).all() and (fin[:, 0, 3] == 255.0).all()


@gpu
def test_largest_deltas_in_every_quadrant(R, oracle, ctx, cases, kernel_sets):
    _, fpc = run_case(R, oracle, ctx, cases, kernel_sets, "corners")
    assert (fpc == 1).all()


@gpu
@pytest.mark.parametrize("voxel", BOUNDARY_VOXELS)
def test_points_on_and_next_to_cell_boundaries(R, oracle, ctx, cases, kernel_sets, voxel):
    run_case(R, oracle, ctx, cases, kernel_sets, f"boundary-{voxel:.4f}")


@gpu
@pytest.mark.parametrize("fused,limit", [("voxel-4", "voxel-above-4"), ("cells-below-32000", "cells-32000")])
def test_admission_boundary(R, oracle, ctx, cases, kernel_sets, fused, limit):
    """voxel 4 m against the next float above it; range_max / voxel one float below 32000 against exactly 32000
    (voxel 2^-10 m, range_max 31.25 m): the same clouds from the fused chain and from the separate passes."""
    a, a_pc = run_case(R, oracle, ctx, cases, kernel_sets, fused)
    b, b_pc = run_case(R, oracle, ctx, cases, kernel_sets, limit)
    assert (a_pc == b_pc).all() and (a_pc > 1).all()
    for s in range(len(a_pc)):
        assert (a[s, : a_pc[s]].view(np.uint32) == b[s, : b_pc[s]].view(np.uint32)).all()


def test_admission_cases_straddle_the_limits():
    v = np.float32(2.0 ** -10)
    below = np.nextafter(np.float32(31.25), np.float32(0.0))
    assert below / v < np.float32(32000.0) == np.float32(31.25) / v
    assert np.nextafter(np.float32(4.0), np.float32(np.inf)) > np.float32(4.0)


@gpu
@pytest.mark.parametrize("k", SOR_KS)
def test_sor_at_every_band(R, oracle, ctx, cases, kernel_sets, k):
    for alpha in (0.0, 1.0, 2.5):
        run_case(R, oracle, ctx, cases, kernel_sets, f"sor-{k}-{alpha}")
    run_case(R, oracle, ctx, cases, kernel_sets, f"sor-{k}-voxel")


@gpu
@pytest.mark.parametrize("stride", [8192, 32768])
def test_large_strides_take_the_separate_passes(R, oracle, ctx, cases, kernel_sets, stride):
    for k in (8, 16, 4):
        run_case(R, oracle, ctx, cases, kernel_sets, f"stride-{stride}-{k}")
