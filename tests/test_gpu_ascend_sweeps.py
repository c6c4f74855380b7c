"""Angle compensation (ascendScanData_) over its whole input domain, bit for bit, on every kernel that writes the
ascended node buffer.

The scans come from the builders of tests/test_ascend_sweep_pieces.py and are built on the device with torch; the
torch restatement there is checked against the numpy one on a sample first and then judges every scan: all 8 bytes of
every ascended node, the status, the slots behind the count (they must keep their sentinel), `path` (0, or the
general kernel exactly where the hand-off rule says), the beam count of every scan, and the ranges, intensities and
angle_increment of a sample of every launch against oracle/scan_oracle.cpp.

Families: A (fill) node 0 measured with key K, every other node unmeasured -- every K at the swept n on the
shared-memory kernel, every 8th K plus the exact-360 keys on scan_fast and the general kernel, every n in 1..8192 with
a few keys, and n 8193..65536 with every 16th key; B (head chain) one measured node at every index f of the swept n,
with the keys around 'clamps at exactly f steps', and every key at f in {1, 2, n/2, n - 1}; C (shared final keys)
measured nodes on computed fill or chain keys, 0..17 of them, Mode A measured duplicates among them.

Kernels: rpl_scan_batch_dev with nodes_out -- the shared-memory EMIT kernel (Mode A and Mode B, bulk-TMA staging at
even strides, plain loads at odd ones), scan_fast_kernel's EMIT variants (RPL_FLAG_NO_SMALL, and strides above 8192)
and scan_general_kernel (RPL_FLAG_FORCE_GENERAL); rpl_scan_views_dev on views that start on odd nodes; rpl_ascend_scan;
and an HQ (0x83) stream session's nodes(apply_ascend=True).  The first launch of every sweep runs once more under the
CUDA profiler, in a child process, to confirm the kernel family it reaches.  Each sweep prints its run time, case
count and peak device memory (-s shows them)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_ascend_sweep_pieces import (CHAIN_NS, KEYS, OK, SENTINEL, SHARED_NS, WIDE_NS, Cases, ascend_words,
                                      chain_cases, chain_every_key_cases, describe, exact360_keys, expected,
                                      extreme_cases, fill_cases, front_keys_every_n, shared_key_cases, spread)
from test_gpu_domain_sweeps import Meter, profiled
from test_gpu_scan_bands import FAST_EMIT_A, FAST_EMIT_B, GENERAL, SMALL

gpu = pytest.mark.gpu

NS, FG = 4, 1          # RPL_FLAG_NO_SMALL, RPL_FLAG_FORCE_GENERAL
SLOTS = 40 << 20       # node slots per launch: inputs, ascended buffer, ranges and intensities ~1 GiB, ~2 GiB at the check
MAX_SCANS = 1 << 17
MAX_DUP_SMALL = 16     # scan_small.cu kMaxDup


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


# ---- the families and the kernels ----------------------------------------------------------------------------------
def family(name, kernel):
    """Lists of Cases (one launch group or more each) of a family, as the kernel runs it"""
    small = kernel == "small"
    if name == "fill every key":
        if small:
            return [fill_cases(n, np.arange(KEYS)) for n in SHARED_NS]
        return ([fill_cases(n, np.union1d(np.arange(0, KEYS, 8), exact360_keys(n))) for n in SHARED_NS]
                + [fill_cases(n, np.union1d(np.arange(0, KEYS, 16), spread(exact360_keys(n), 512))) for n in WIDE_NS])
    if name == "fill every n":
        return [Cases.cat([fill_cases(n, front_keys_every_n(n)) for n in range(lo, min(lo + 64, 8193))])
                for lo in range(1, 8193, 64)]
    if name == "head chain":
        return ([chain_cases(n) for n in CHAIN_NS]
                + [chain_every_key_cases(n, 1 if small else 8) for n in (360, 3200, 8192)])
    return [shared_key_cases(), extreme_cases()]


FAMILIES = ["fill every key", "fill every n", "head chain", "shared keys"]
KERNELS = {  # name: (flags, kernel of Mode A, kernel of Mode B; None: the general kernel alone)
    "small": (0, SMALL, SMALL),
    "fast": (NS, FAST_EMIT_A, FAST_EMIT_B),
    "general": (FG, None, None),
}


def stride_of(kernel, n, g):
    """the small kernel stages even strides with one bulk copy and odd ones with plain loads; scan_fast reads odd
    strides 8 bytes off a 16-byte boundary in every second scan"""
    n = np.asarray(n, np.int64)
    even = n + (n & 1)
    if kernel == "small":
        return even if g % 2 == 0 else np.where(n >= 8192, even, n | 1)
    return np.where((g % 2 == 1) & (n < KEYS), n | 1, even)


def groups(cases_list, kernel):
    """(Cases, stride) launch groups: at most SLOTS node slots and MAX_SCANS scans, scans of one stride"""
    g = 0
    for c in cases_list:
        c = c.take(np.argsort(c.n, kind="stable"))
        i = 0
        while i < len(c):
            top = c.n[i:i + MAX_SCANS]
            ok = np.arange(1, len(top) + 1) * stride_of(kernel, top, g) <= SLOTS
            j = i + (len(top) if ok.all() else max(1, int(np.argmin(ok))))
            yield c.take(np.arange(i, j)), int(stride_of(kernel, c.n[j - 1], g)), g
            g += 1
            i = j


def want_path(kernel, d, dm, counts, mode_a, anym):
    if kernel == "general":
        return torch.ones_like(d)
    if kernel == "fast":
        p = d > 0
    else:
        p = (d > MAX_DUP_SMALL) | ((dm > 0) & (not mode_a))
    return torch.where(anym, p.to(torch.int64), torch.zeros_like(d))


def shared(words, counts, live, srt):
    """(D, DM): nodes beyond the first of their final key, measured nodes beyond the first of their key"""
    sk = srt >> 17
    d = live.sum(1) - (((sk[:, 1:] != sk[:, :-1]) & live[:, 1:]).sum(1) + live[:, 0].to(torch.int64))
    meas = live & (((words >> 16) & 0xFFFFFFFF) != 0)
    mk = torch.where(meas, words & 0xFFFF, torch.full_like(words, KEYS)).sort(1).values
    dm = meas.sum(1) - (((mk[:, 1:] != mk[:, :-1]) & (mk[:, 1:] < KEYS)).sum(1) + (mk[:, 0] < KEYS).to(torch.int64))
    return d, dm, meas.sum(1)


def outputs(S, stride, dev):
    o = dict(nodes_out=torch.full((S, stride), SENTINEL, dtype=torch.int64, device=dev),
             ranges=torch.full((S, stride), float("nan"), device=dev),
             intensities=torch.full((S, stride), float("nan"), device=dev),
             beam_counts=torch.full((S,), -1, dtype=torch.int32, device=dev),
             angle_increment=torch.full((S,), float("nan"), device=dev),
             status=torch.full((S,), -1, dtype=torch.int32, device=dev),
             path=torch.full((S,), -1, dtype=torch.int32, device=dev))
    return o, {k: v.data_ptr() for k, v in o.items()}


def launch(R, ctx, words, counts32, stride, params):
    o, ptrs = outputs(words.shape[0], stride, words.device)
    torch.cuda.synchronize()  # the buffers were filled on torch's stream; the library runs on its own
    ctx.scan_batch_dev(words.data_ptr(), counts32.data_ptr(), words.shape[0], stride, params, **ptrs)
    ctx.synchronize()
    torch.cuda.synchronize()
    return o


def judge(words, counts):
    """what every launch of these scans must give: (status, ascended words, D, DM, measured nodes) per scan"""
    st, want, _, live, srt = expected(words, counts)
    d, dm, m = shared(words, counts, live, srt)
    del live, srt
    return st, want, d, dm, m


def check_launch(O, o, words, counts, jd, kernel, mode_a, newp, what, n_sample=3):
    """the ascended buffers, statuses and paths of every scan; beam counts of every scan; ranges, intensities and
    angle_increment of a sample against the oracle, and nothing written behind the beam count"""
    S, W = words.shape
    st, want, d, dm, m = jd
    where = _mismatch(o["nodes_out"], o["status"], st, want)
    if where is not None:
        pytest.fail(f"{what}: {describe(where, words, counts)}")
    wp = want_path(kernel, d, dm, counts, mode_a, st == OK)
    bad = (o["path"].to(torch.int64) != wp).nonzero()
    assert bad.numel() == 0, f"{what}: scan {int(bad[0])} (n {int(counts[bad[0]])}, D {int(d[bad[0]])}, measured " \
                             f"duplicates {int(dm[bad[0]])}): path {int(o['path'][bad[0]])}, want {int(wp[bad[0]])}"
    bad = (o["beam_counts"].to(torch.int64) != m).nonzero()
    assert bad.numel() == 0, f"{what}: scan {int(bad[0])}: beam_count {int(o['beam_counts'][bad[0]])}, want {int(m[bad[0]])}"
    col = torch.arange(W, device=words.device)[None, :]
    behind = col >= m[:, None]
    assert bool((torch.isnan(o["ranges"]) | ~behind).all() and (torch.isnan(o["intensities"]) | ~behind).all()), \
        f"{what}: a LaserScan slot written behind the beam count"
    rng = np.random.default_rng(S * 7 + W)
    pick = set([0, S - 1] + rng.integers(0, S, n_sample).tolist())
    dup = (d > 0).nonzero()
    if dup.numel():
        pick.add(int(dup[0]))
    prm = O.scan_params(newp, int(mode_a), 0, 1)
    w_host = words.cpu().numpy() if S * W < (1 << 22) else None
    for s in sorted(pick):
        n = int(counts[s])
        row = (w_host[s] if w_host is not None else words[s].cpu().numpy())[:n]
        hdr, r, it = O.publish(np.ascontiguousarray(row).view(O.NODE_DTYPE), prm, stable=True)
        k = int(hdr.beam_count)
        assert k == int(o["beam_counts"][s]), (what, s)
        got_r, got_i = o["ranges"][s, :k].cpu().numpy(), o["intensities"][s, :k].cpu().numpy()
        assert got_r.tobytes() == r.tobytes() and got_i.tobytes() == it.tobytes(), f"{what}: scan {s} LaserScan"
        if k:
            assert np.float32(hdr.angle_increment).tobytes() == o["angle_increment"][s].cpu().numpy().tobytes(), (what, s)
    return int((d > 0).sum()), int((wp > 0).sum())


def _mismatch(got, status, want_st, want):
    status = status.to(torch.int64) & 0xFFFFFFFF  # (a u32 read through int32)
    bad = (status != want_st).nonzero()
    if bad.numel():
        s = int(bad[0])
        return s, -1, int(status[s]), int(want_st[s])
    ok = got == want
    if bool(ok.all()):
        return None
    s, j = (int(v) for v in (~ok).nonzero()[0])
    return s, j, int(got[s, j]), int(want[s, j])


def mode_of(g, kernel):
    """(Mode A, new protocol) of launch group g: the general kernel alternates, the others run both modes"""
    return [(g % 2 == 1, (g >> 1) & 1)] if kernel == "general" else [(False, g & 1), (True, (g + 1) & 1)]


def max_stride(cases_list, kernel):
    return max(int(stride_of(kernel, c.n.max(), g)) for c in cases_list for g in (0, 1))


# ---- the profiled first launches -------------------------------------------------------------------------------------
def first_launch_kernels():
    """{case: sorted kernels that ran} for the first launch group of every (family, kernel, mode), each under the
    CUDA profiler (run by kernels_in_a_child_process)."""
    import rplidar_ros2_driver_b200 as R

    dev = torch.device("cuda")
    seen = {}
    for fam in FAMILIES:
        for kernel, (flags, ka, kb) in KERNELS.items():
            c, stride, g = next(groups(family(fam, kernel), kernel))
            c = c.take(np.arange(min(len(c), 256)))
            words = c.words(stride, dev)
            counts32 = torch.as_tensor(c.n, device=dev).to(torch.int32)
            for mode_a, newp in mode_of(0, kernel) if kernel != "general" else [(False, 0)]:
                with R.Context(0, stride, len(c)) as ctx:
                    want = {ka if mode_a else kb, GENERAL} - {None}
                    seen[f"{fam} {kernel} {int(mode_a)}"] = profiled(
                        lambda: launch(R, ctx, words, counts32, stride, R.scan_params(newp, int(mode_a), 0, 1, flags)),
                        ctx, want)
    return {k: sorted(v) for k, v in seen.items()}


def kernels_in_a_child_process():
    """As tests/test_gpu_domain_sweeps.py: the profiler runs in a Python process of its own, which takes its CUDA
    activity tracing state with it when it exits."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"),
                                                       os.environ.get("PYTHONPATH", "")]))
    code = ("import json, test_gpu_ascend_sweeps as T; "
            "print('KERNELS ' + json.dumps(T.first_launch_kernels()), flush=True)")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, env=env, capture_output=True, text=True,
                       timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")]
    assert r.returncode == 0 and lines, f"the profiling process failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return {k: set(v) for k, v in json.loads(lines[-1][len("KERNELS "):]).items()}


@pytest.fixture(scope="module")
def kernels_seen():
    return kernels_in_a_child_process()


# ---- the tests -------------------------------------------------------------------------------------------------------
@gpu
def test_torch_restatement_on_the_device_equals_numpy():
    dev = torch.device("cuda")
    rng = np.random.default_rng(11)
    parts = [fill_cases(n, rng.choice(KEYS, 40, replace=False)) for n in SHARED_NS]
    parts += [fill_cases(n, exact360_keys(n)[:20]) for n in SHARED_NS if len(exact360_keys(n))]
    parts += [chain_cases(n).take(rng.choice(len(chain_cases(n)), 60, replace=False)) for n in (17, 360, 3200)]
    parts += [shared_key_cases(), extreme_cases()]
    c = Cases.cat(parts)
    W = int(c.n.max())
    words = c.words(W)
    st, out = ascend_words(words, c.n)
    assert (c.words(W, dev).cpu().numpy() == words).all()  # the device builder builds the same scans
    t_st, t_out, *_ = expected(torch.from_numpy(words).to(dev), torch.from_numpy(c.n).to(dev))
    assert (t_st.cpu().numpy() == st).all() and (t_out.cpu().numpy() == out).all()


@gpu
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("fam", FAMILIES)
def test_ascended_buffer_over_the_domain(R, oracle, kernels_seen, fam, kernel):
    flags, ka, kb = KERNELS[kernel]
    for mode_a, _ in mode_of(0, kernel) if kernel != "general" else [(False, 0)]:
        assert kernels_seen[f"{fam} {kernel} {int(mode_a)}"] == {ka if mode_a else kb, GENERAL} - {None}, kernels_seen
    dev = torch.device("cuda")
    cases_list = family(fam, kernel)
    meter = Meter()
    n_scans = n_nodes = n_dup = n_general = 0
    with meter.context(R, max_stride(cases_list, kernel), MAX_SCANS) as ctx:
        for c, stride, g in groups(cases_list, kernel):
            words = c.words(stride, dev, first_scan=g)
            counts = torch.as_tensor(c.n, device=dev)
            counts32 = counts.to(torch.int32)
            jd = judge(words, counts)
            for mode_a, newp in mode_of(g, kernel):
                what = (f"{fam} on {kernel} (Mode {'A' if mode_a else 'B'}, stride {stride}, flags {flags}, "
                        f"n {int(c.n.min())}..{int(c.n.max())})")
                o = launch(R, ctx, words, counts32, stride, R.scan_params(newp, int(mode_a), 0, 1, flags))
                nd, ng = check_launch(oracle, o, words, counts, jd, kernel, mode_a, newp, what)
                n_scans += len(c)
                n_nodes += int(c.n.sum())
                n_dup, n_general = n_dup + nd, n_general + ng
                del o
            del words, jd
    if fam == "shared keys" and kernel != "general":
        assert n_dup >= 30 and n_general >= 2
    meter.report(f"ascend {fam} on {kernel}",
                 f"{n_scans} scans ({n_nodes} nodes; {n_dup} with shared final keys, {n_general} handed on)")


@gpu
def test_views_on_odd_first_nodes(R, oracle):
    """rpl_scan_views_dev with nodes_out: every view starts on an odd node (the bulk copy starts one node early), the
    last one ends at the end of the buffer (its rounded copy would run past it: plain loads)"""
    dev = torch.device("cuda")
    rng = np.random.default_rng(23)
    parts = [shared_key_cases(), extreme_cases()]
    parts += [fill_cases(n, exact360_keys(n)[:8]) for n in SHARED_NS if len(exact360_keys(n))]
    parts += [chain_cases(n).take(rng.choice(len(chain_cases(n)), 40, replace=False)) for n in (33, 360, 8192)]
    c = Cases.cat(parts)
    stride = 8192
    words = c.words(stride, dev)
    first, at = [], 1
    for n in c.n.tolist():
        at += 1 - (at & 1) if n else 0
        first.append(at)
        at += n
    total = at
    flat = torch.zeros(total + (total & 1), dtype=torch.int64, device=dev)
    col = torch.arange(stride, device=dev)[None, :]
    live = col < torch.as_tensor(c.n, device=dev)[:, None]
    idx = (torch.as_tensor(first, device=dev)[:, None] + col)[live]
    flat[idx] = words[live]
    views = torch.as_tensor(np.stack([first, c.n], 1).astype(np.int32), device=dev)
    counts = torch.as_tensor(c.n, device=dev)
    jd = judge(words, counts)
    assert first[-1] % 2 == 1 and first[-1] + int(c.n[-1]) == total
    with R.Context(0, stride, len(c)) as ctx:
        for mode_a in (False, True):
            o, ptrs = outputs(len(c), stride, dev)
            torch.cuda.synchronize()
            ctx.scan_views_dev(flat.data_ptr(), total, views.data_ptr(), len(c), stride,
                               R.scan_params(1, int(mode_a), 0, 1), **ptrs)
            ctx.synchronize()
            torch.cuda.synchronize()
            check_launch(oracle, o, words, counts, jd, "small", mode_a, 1, f"views (Mode {'A' if mode_a else 'B'})", 8)
    print(f"\n[ascend sweep] views: {len(c)} scans on odd first nodes, on {torch.cuda.get_device_name()}")


@gpu
def test_single_scan_ascend(R):
    """rpl_ascend_scan, in place on host buffers, on a sample of every family, the widest scans included"""
    rng = np.random.default_rng(29)
    parts = [shared_key_cases().take(np.arange(0, 200, 7)), extreme_cases()]
    parts += [fill_cases(n, np.concatenate([exact360_keys(n)[:2], rng.integers(0, KEYS, 2)])) for n in SHARED_NS + WIDE_NS]
    parts += [chain_cases(n).take(rng.choice(len(chain_cases(n)), 10, replace=False)) for n in (9, 360, 8192)]
    c = Cases.cat(parts)
    with R.Context(0, KEYS, 1) as ctx:
        for s in range(len(c)):
            one = c.take([s])
            n = int(one.n[0])
            w = one.words(n)
            rc, buf = ctx.ascend_scan(np.ascontiguousarray(w[0]).view(R.NODE_DTYPE))
            st, want = ascend_words(w, one.n)
            got = buf.view(np.int64)
            assert rc == st[0], (s, n, hex(rc))
            bad = np.flatnonzero(got != want[0])
            assert not len(bad), describe((0, int(bad[0]), int(got[bad[0]]), int(want[0, bad[0]])), w, one.n)


@gpu
def test_session_nodes_of_an_hq_stream(R, oracle):
    """An HQ (0x83) capsule stream session's nodes(apply_ascend=True) -- the grab_scan_data buffers, ascended by the
    EMIT launch with out_first placement -- over revolutions of the families: every buffer equals the restatement"""
    from test_gpu_stream_cloud import Feed
    from test_gpu_stream_nodes import crafted_stream, run

    O = oracle
    rng = np.random.default_rng(31)
    sc = shared_key_cases()
    parts = [sc.take(rng.choice(len(sc), 24, replace=False)), extreme_cases().take([3, 5, 6, 8, 9])]
    parts += [fill_cases(n, exact360_keys(n)[:2]) for n in (360, 1000, 3200, 8191)]
    parts += [chain_cases(n).take(rng.choice(len(chain_cases(n)), 4, replace=False)) for n in (40, 360, 3200)]
    c = Cases.cat(parts)
    revs = []
    for s in range(len(c)):
        n = int(c.n[s])
        r = np.ascontiguousarray(c.take([s]).words(n)[0]).view(O.NODE_DTYPE).copy()
        r["flag"] = 2
        r["flag"][0] = 1  # the start flag opens the revolution
        revs.append(r)
    d = crafted_stream(O, revs)
    feed = Feed(R, O, "framed", 0x83)
    with R.Context(0, 8192, 64) as ctx:
        with feed.session(ctx, 1, len(d), 8192, 64) as sess:
            _, rows = run(R, feed, sess, [[d]], len(d), dict(apply_ascend=True))
    got = rows[0][1:]  # behind the leading revolution crafted_stream puts first
    assert len(got) == len(revs)
    for s, (r, (rc, b)) in enumerate(zip(revs, got)):
        st, want = ascend_words(r.view(np.int64)[None], [len(r)])
        assert rc == st[0] and b == want[0].tobytes(), f"session revolution {s} (n {len(r)})"
