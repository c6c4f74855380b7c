"""Calls of one context issued back to back on different streams, with nothing ordering them but the library: the
device calls run their scan kernels on lane 0's scan scratch (fallback list and count, general- and fast-kernel
workspaces, the post passes' cloud workspace), whatever stream they come on, and take turns on it.  Every case issues
two calls on their own torch streams, each stream waiting on one event recorded after a sleep on a third stream so
that the calls start together, and compares every output bit for bit with the same calls issued one at a time on the
same context; a sample is compared with the oracle.  Half of each batch's scans carry duplicated measured keys, so
that the general kernel and the fallback list run in every case.

Each case runs on a fresh context whose max_scans holds every scan issued at once, with the concurrent batches of one
size and no earlier call larger: calls that did not take turns would give wrong results, never touch memory outside
their buffers."""
import numpy as np
import pytest

from test_capsule_bytes_pieces import raw_stream
from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_stream import _check_oracle, _scans
from test_gpu_scan_bands import oracle_scans
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu

GATE = 20_000_000   # cycles slept before the gate opens (about 10 ms)
SHORT = 2_000_000   # host-call cases: the host call's copies start while the gate is shut
PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend
WINDOW = dict(range_min=0.15, range_max=40.0)
SOR_VOXEL = dict(sor_k=8, sor_alpha=1.0, voxel_size=0.05)


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


# ---- running calls at once and one at a time -----------------------------------------------------------------------
# A call is make() -> (issue, fetch, host): issue(stream handle) enqueues it (a host call ignores the handle and
# returns when it is done), fetch() returns its outputs as numpy arrays once everything is synchronised.
def run_gated(torch, ctx, calls, sleep):
    torch.cuda.synchronize()
    gate = torch.cuda.Stream()
    streams = [torch.cuda.Stream() for _ in calls]
    with torch.cuda.stream(gate):
        torch.cuda._sleep(sleep)
    opened = torch.cuda.Event()
    opened.record(gate)
    for st, (issue, _, host) in zip(streams, calls):
        if not host:
            st.wait_event(opened)
            issue(st.cuda_stream)
    for issue, _, host in calls:  # host calls while the device calls wait for the gate or run
        if host:
            issue(None)
    ctx.synchronize()
    torch.cuda.synchronize()
    return [fetch() for _, fetch, _ in calls]


def run_serial(torch, ctx, calls):
    for issue, _, _ in calls:
        torch.cuda.synchronize()
        issue(torch.cuda.Stream().cuda_stream)
        ctx.synchronize()
        torch.cuda.synchronize()
    return [fetch() for _, fetch, _ in calls]


def run_both(torch, ctx, makes, sleep=GATE):
    """the calls gated onto streams of their own, then the same calls (fresh outputs) one at a time: both must agree
    bit for bit.  Returns the outputs of both runs."""
    conc = run_gated(torch, ctx, [m() for m in makes], sleep)
    ser = run_serial(torch, ctx, [m() for m in makes])
    for i, (a, b) in enumerate(zip(conc, ser)):
        assert a.keys() == b.keys()
        for k in a:
            ga, gb = np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)
            assert ga.shape == gb.shape and (ga == gb).all(), f"call {i}: {k} differs from the call issued alone"
    return conc, ser


def host_of(t):
    return t.cpu().numpy()


# ---- inputs ----------------------------------------------------------------------------------------------------------
def dup_batch(O, n, stride, seed):
    """n scans of `stride` measured nodes, keys distinct but in the odd scans, where 24 measured keys appear twice:
    more than the shared-memory kernel places itself, so that those scans go to the general kernel"""
    nodes = O.synth_batch(seed, n, stride, 1).copy()
    d = nodes["dist_mm_q2"]
    d[d == 0] = 4321
    rng = np.random.default_rng(seed)
    for s in range(1, n, 2):
        at = rng.choice(stride, 48, replace=False)
        nodes["angle_z_q14"][s, at[24:]] = nodes["angle_z_q14"][s, at[:24]]
    counts = np.full(n, stride, np.uint32)
    counts[::3] -= np.arange(len(counts[::3]), dtype=np.uint32) % 97  # ragged counts as well
    return nodes, counts


def to_dev(torch, R, nodes, counts):
    return (torch.from_numpy(nodes.view(np.uint8).reshape(nodes.shape[0], -1)).cuda(),
            torch.from_numpy(counts.view(np.int32)).cuda())


# ---- the calls -------------------------------------------------------------------------------------------------------
def scan_dev(torch, R, ctx, nodes_t, counts_t, n, stride, emit=False):
    def make():
        o = dict(ranges=torch.full((n, stride), float("nan"), device="cuda"),
                 intensities=torch.full((n, stride), float("nan"), device="cuda"),
                 **{k: torch.full((n,), -1, dtype=torch.int32, device="cuda") for k in ("beams", "status", "path")},
                 inc=torch.full((n,), float("nan"), device="cuda"))
        if emit:
            o["nodes"] = nodes_t.clone()  # the kernels write only the scans they ascend

        def issue(st):
            ctx.scan_batch_dev(nodes_t.data_ptr(), counts_t.data_ptr(), n, stride, R.scan_params(*PARAMS),
                               nodes_out=o["nodes"].data_ptr() if emit else None, ranges=o["ranges"].data_ptr(),
                               intensities=o["intensities"].data_ptr(), beam_counts=o["beams"].data_ptr(),
                               angle_increment=o["inc"].data_ptr(), status=o["status"].data_ptr(),
                               path=o["path"].data_ptr(), stream=st)

        return issue, lambda: {k: host_of(v) for k, v in o.items()}, False

    return make


def scan_host(R, ctx, nodes, counts):
    def make():
        o = {}

        def issue(_):
            out = ctx.scan_batch(nodes, counts, R.scan_params(*PARAMS))
            o.update(ranges=out["ranges"], intensities=out["intensities"], beams=out["beam_counts"].view(np.int32),
                     status=out["status"].view(np.int32), path=out["path"].view(np.int32), inc=out["angle_increment"])

        return issue, lambda: dict(o), True

    return make


def trimmed(xyzi, pc):
    """clouds as compared: each scan's points up to its count (the rows behind it are scratch)"""
    xyzi = xyzi.copy()
    for j, k in enumerate(pc.view(np.uint32)):
        xyzi[j, k:] = 0
    return dict(xyzi=xyzi, point_counts=pc)


def cloud_dev(torch, R, ctx, nodes_t, counts_t, n, stride, flags):
    def make():
        xyzi = torch.full((n, stride, 4), float("nan"), device="cuda")
        pc = torch.full((n,), -1, dtype=torch.int32, device="cuda")

        def issue(st):
            ctx.cloud_batch_dev(nodes_t.data_ptr(), counts_t.data_ptr(), n, stride,
                                R.cloud_params(flags=flags, is_new_protocol=1, **WINDOW, **SOR_VOXEL), xyzi.data_ptr(),
                                pc.data_ptr(), stream=st)

        return issue, lambda: trimmed(host_of(xyzi), host_of(pc)), False

    return make


def cloud_host(R, ctx, nodes, counts, flags):
    def make():
        o = {}

        def issue(_):
            xyzi, pc = ctx.cloud_batch(nodes, counts, R.cloud_params(flags=flags, is_new_protocol=1, **WINDOW,
                                                                     **SOR_VOXEL))
            o.update(trimmed(xyzi, pc.view(np.int32)))

        return issue, lambda: dict(o), True

    return make


def check_scans_vs_oracle(O, nodes, counts, got, which):
    exp = oracle_scans(O, nodes[which].copy(), counts[which], *PARAMS)
    for i, s in enumerate(which):
        m = int(exp["beam_counts"][i])
        assert int(got["beams"][s]) == m, s
        assert (got["ranges"][s, :m].view(np.uint32) == exp["ranges"][i, :m].view(np.uint32)).all(), s
        assert (got["intensities"][s, :m].view(np.uint32) == exp["intensities"][i, :m].view(np.uint32)).all(), s


def check_clouds_vs_oracle(O, nodes, counts, got, which):
    for s in which:
        e = O.cloud(nodes[s, : counts[s]], O.cloud_params(is_new_protocol=1, **WINDOW, **SOR_VOXEL))
        assert int(got["point_counts"][s]) == e.shape[0], s
        assert (got["xyzi"][s, : e.shape[0]].view(np.uint32) == e.view(np.uint32)).all(), s


SAMPLE = [0, 1, 2, 3, 6, 7]


# ---- scan batches --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stride,emit", [(4096, False), (12288, True)], ids=["mode-b-small", "fast-ascended"])
def test_two_scan_batches(R, oracle, torch, stride, emit):
    """two rpl_scan_batch_dev: Mode B in the shared-memory kernel, or above 8192 nodes with the ascended buffer
    (scan_fast_kernel and its workspace); the duplicate-key scans then go through the fallback list to the general
    kernel"""
    n = 512 if stride <= 8192 else 128
    ctx = R.Context(0, stride, 2 * n)
    data = [dup_batch(oracle, n, stride, 11 + i) for i in range(2)]
    dev = [to_dev(torch, R, *d) for d in data]
    conc, ser = run_both(torch, ctx, [scan_dev(torch, R, ctx, *t, n, stride, emit) for t in dev])
    for (nodes, counts), got in zip(data, conc):
        assert (got["path"] == np.arange(n) % 2).all()  # the odd scans went to the general kernel
        check_scans_vs_oracle(oracle, nodes, counts, got, SAMPLE)
    ctx.close()


def test_scan_batch_host_call_meets_a_device_call(R, oracle, torch):
    """rpl_scan_batch (lane 0's stream) while a gated rpl_scan_batch_dev waits on a caller stream"""
    n, stride = 512, 4096
    ctx = R.Context(0, stride, n)
    (n0, c0), (n1, c1) = dup_batch(oracle, n, stride, 21), dup_batch(oracle, n, stride, 22)
    conc, _ = run_both(torch, ctx, [scan_dev(torch, R, ctx, *to_dev(torch, R, n0, c0), n, stride),
                                    scan_host(R, ctx, n1, c1)], sleep=SHORT)
    for (nodes, counts), got in zip(((n0, c0), (n1, c1)), conc):
        assert (got["path"] == np.arange(n) % 2).all()
        check_scans_vs_oracle(oracle, nodes, counts, got, SAMPLE)
    ctx.close()


# ---- PointCloud2 batches ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "no-fused"])
def test_two_cloud_batches(R, oracle, torch, fused):
    """two rpl_cloud_batch_dev with SOR and the voxel grid: fused into the shared-memory kernel (the duplicate-key scans
    through the general kernel to the list-restricted post passes), or RPL_CLOUD_NO_FUSED (post passes over every
    scan on lane 0's cloud workspace)"""
    n, stride = 256, 4096
    flags = 0 if fused else R.CLOUD_NO_FUSED
    ctx = R.Context(0, stride, 2 * n)
    data = [dup_batch(oracle, n, stride, 31 + i) for i in range(2)]
    conc, _ = run_both(torch, ctx, [cloud_dev(torch, R, ctx, *to_dev(torch, R, *d), n, stride, flags) for d in data])
    for (nodes, counts), got in zip(data, conc):
        check_clouds_vs_oracle(oracle, nodes, counts, got, SAMPLE)
    ctx.close()


def test_cloud_host_call_meets_a_device_call(R, oracle, torch):
    n, stride = 256, 4096
    ctx = R.Context(0, stride, n)
    (n0, c0), (n1, c1) = dup_batch(oracle, n, stride, 41), dup_batch(oracle, n, stride, 42)
    conc, _ = run_both(torch, ctx, [cloud_dev(torch, R, ctx, *to_dev(torch, R, n0, c0), n, stride, 0),
                                    cloud_host(R, ctx, n1, c1, 0)], sleep=SHORT)
    for (nodes, counts), got in zip(((n0, c0), (n1, c1)), conc):
        check_clouds_vs_oracle(oracle, nodes, counts, got, SAMPLE)
    ctx.close()


# ---- sessions --------------------------------------------------------------------------------------------------------
N_STREAMS, MAX_NODES, MAX_SCANS = 8, 4096, 32
ULTRA_CAPS = 400  # about 13 revolutions of ultra capsules per stream


class Session:
    """a session kind and its input: 'framed' ultra capsules, 'stamped' (push_ts_dev) or 'bytes' (push_bytes_dev)"""

    def __init__(self, R, O, ctx, kind, seed, ans=0x84):
        self.R, self.ctx, self.kind, self.ans = R, ctx, kind, ans
        n = N_STREAMS
        if kind == "bytes":
            self.data = [raw_stream(O, ans, seed + s) for s in range(n)]
            self.stride = max(len(b) for b in self.data)
            self.buf = np.full((n, self.stride), 0xEE, np.uint8)
        else:
            self.data = [format_stream(O, ans, ULTRA_CAPS, seed + s, sync_every=97 + s if s % 2 else None)
                         for s in range(n)]
            self.stride = ULTRA_CAPS
            self.buf = np.zeros((n, ULTRA_CAPS, O.capsule_bytes(ans)), np.uint8)
        self.cnt = np.zeros(n, np.uint32)
        for s, d in enumerate(self.data):
            self.buf[s, : len(d)] = d
            self.cnt[s] = len(d)
        rng = np.random.default_rng(seed)
        self.rx = (10_000_000 + np.cumsum(rng.integers(200, 3000, (n, self.stride)), axis=1)).astype(np.uint64)
        self.opened = []

    def open(self):
        R, n = self.R, N_STREAMS
        if self.kind == "bytes":
            sess = R.CapsuleByteStreamSession(self.ctx, self.ans, n, self.stride, MAX_NODES, MAX_SCANS)
        else:
            sess = R.CapsuleStreamSession(self.ctx, self.ans, n, self.stride, MAX_NODES, MAX_SCANS)
        self.opened.append(sess)
        return sess

    def push_dev(self, torch, pushed=None):
        """make() of one session's push_dev of the whole streams, on a fresh session (pushed: the list it is put in)"""
        R, n, NS = self.R, N_STREAMS, N_STREAMS * MAX_SCANS

        def make():
            sess = self.open()
            if pushed is not None:
                pushed.append(sess)
            d_buf, d_cnt = torch.from_numpy(self.buf).cuda(), torch.from_numpy(self.cnt.view(np.int32)).cuda()
            d_rx = torch.from_numpy(self.rx.view(np.int64)).cuda()
            o = dict(ranges=torch.full((NS, MAX_NODES), -1.0, device="cuda"),
                     intensities=torch.full((NS, MAX_NODES), -1.0, device="cuda"),
                     beam_counts=torch.zeros(NS, dtype=torch.int32, device="cuda"),
                     angle_increment=torch.zeros(NS, device="cuda"),
                     scans_per_stream=torch.zeros(n, dtype=torch.int32, device="cuda"),
                     scan_begin_ts_us=torch.full((NS,), -1, dtype=torch.int64, device="cuda"))
            args = (d_buf.data_ptr(), d_cnt.data_ptr(), R.scan_params(*PARAMS)) + tuple(
                o[k].data_ptr() for k in ("ranges", "intensities", "beam_counts", "angle_increment", "scans_per_stream"))

            def issue(st):
                if self.kind == "framed":
                    sess.push_dev(*args, stream=st)
                elif self.kind == "stamped":
                    sess.push_dev(*args, stream=st, rx_us=d_rx.data_ptr(), timing=R.Timing(*TIMINGS[0]),
                                  scan_begin_ts_us=o["scan_begin_ts_us"].data_ptr())
                else:
                    sess.push_dev(*args, stream=st)

            def fetch():
                got = {k: host_of(v) for k, v in o.items()}
                for k in ("beam_counts", "scans_per_stream"):
                    got[k] = got[k].view(np.uint32)
                return got

            keep = (d_buf, d_cnt, d_rx)  # alive until fetched
            return issue, lambda: (keep, fetch())[1], False

        return make

    def push_host(self):
        R = self.R

        def make():
            sess = self.open()
            o = {}

            def issue(_):
                o.update(sess.push(self.buf, self.cnt, R.scan_params(*PARAMS)))

            return issue, lambda: dict(o), True

        return make

    def close(self):
        for s in self.opened:
            s.close()


def check_session_oracle(O, sess, got):
    if sess.kind == "framed":
        _check_oracle(O, sess.ans, _scans(got, N_STREAMS, MAX_SCANS), sess.data, MAX_NODES, [0, 3, 5])


@pytest.mark.parametrize("kind", ["framed", "stamped", "bytes"], ids=["push_dev", "push_ts_dev", "push_bytes_dev"])
def test_two_session_pushes(R, oracle, torch, kind):
    """two ultra sessions' device pushes on two streams: the decoder and the assembler take turns on the assemble
    scratch, the scan kernels on lane 0's scan scratch"""
    ctx = R.Context(0, MAX_NODES, 2 * N_STREAMS * MAX_SCANS)
    sessions = [Session(R, oracle, ctx, kind, 500 + 50 * i) for i in range(2)]
    conc, _ = run_both(torch, ctx, [s.push_dev(torch) for s in sessions])
    for s, got in zip(sessions, conc):
        assert (got["scans_per_stream"] >= 5).all() and (got["scans_per_stream"] <= MAX_SCANS).all()
        check_session_oracle(oracle, s, got)
        s.close()
    ctx.close()


def test_session_host_push_meets_a_device_push(R, oracle, torch):
    ctx = R.Context(0, MAX_NODES, 2 * N_STREAMS * MAX_SCANS)
    sessions = [Session(R, oracle, ctx, "framed", 600 + 50 * i) for i in range(2)]
    conc, _ = run_both(torch, ctx, [sessions[0].push_dev(torch), sessions[1].push_host()], sleep=SHORT)
    for s, got in zip(sessions, conc):
        check_session_oracle(oracle, s, got)
        s.close()
    ctx.close()


def test_scan_views_meet_a_session_push(R, oracle, torch):
    """rpl_scan_views_dev over a batch of views of the session's scan count and stride, against a session push_dev"""
    ns, stride = N_STREAMS * MAX_SCANS, MAX_NODES
    ctx = R.Context(0, MAX_NODES, 2 * ns)
    nodes, counts = dup_batch(oracle, ns, stride, 71)
    nodes_t = torch.from_numpy(nodes.view(np.uint8).reshape(-1)).cuda()
    views = np.stack([np.arange(ns, dtype=np.uint32) * stride, counts], axis=1)
    views_t = torch.from_numpy(views.view(np.int32)).cuda()
    sess = Session(R, oracle, ctx, "framed", 700)

    def views_call():
        o = dict(ranges=torch.full((ns, stride), float("nan"), device="cuda"),
                 intensities=torch.full((ns, stride), float("nan"), device="cuda"),
                 beams=torch.full((ns,), -1, dtype=torch.int32, device="cuda"),
                 path=torch.full((ns,), -1, dtype=torch.int32, device="cuda"),
                 inc=torch.full((ns,), float("nan"), device="cuda"))

        def issue(st):
            ctx.scan_views_dev(nodes_t.data_ptr(), ns * stride, views_t.data_ptr(), ns, stride, R.scan_params(*PARAMS),
                               ranges=o["ranges"].data_ptr(), intensities=o["intensities"].data_ptr(),
                               beam_counts=o["beams"].data_ptr(), angle_increment=o["inc"].data_ptr(),
                               path=o["path"].data_ptr(), stream=st)

        return issue, lambda: {k: host_of(v) for k, v in o.items()}, False

    conc, _ = run_both(torch, ctx, [views_call, sess.push_dev(torch)])
    assert (conc[0]["path"] == np.arange(ns) % 2).all()
    check_scans_vs_oracle(oracle, nodes, counts, conc[0], SAMPLE)
    check_session_oracle(oracle, sess, conc[1])
    sess.close()
    ctx.close()


def test_session_cloud_meets_a_cloud_batch(R, oracle, torch):
    """a session's cloud_dev (after a push of its own) against an rpl_cloud_batch_dev of its scan count and stride"""
    ns, stride = N_STREAMS * MAX_SCANS, MAX_NODES
    ctx = R.Context(0, MAX_NODES, 2 * ns)
    nodes, counts = dup_batch(oracle, ns, stride, 81)
    sess = Session(R, oracle, ctx, "framed", 800)
    pushed = []
    prm = R.cloud_params(is_new_protocol=1, **WINDOW, **SOR_VOXEL)

    def session_cloud():
        issue_push, fetch_push, _ = sess.push_dev(torch, pushed)()
        issue_push(None)  # the push, on the context's stream, before the gate
        ctx.synchronize()
        fetch_push()
        xyzi = torch.full((ns, MAX_NODES, 4), float("nan"), device="cuda")
        pc = torch.full((ns,), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

        def issue(st):
            pushed[-1].cloud_dev(prm, xyzi.data_ptr(), pc.data_ptr(), stream=st)

        return issue, lambda: trimmed(host_of(xyzi), host_of(pc)), False

    conc, _ = run_both(torch, ctx, [session_cloud, cloud_dev(torch, R, ctx, *to_dev(torch, R, nodes, counts), ns,
                                                             stride, 0)])
    assert (conc[0]["point_counts"] > 0).sum() >= N_STREAMS * 8
    check_clouds_vs_oracle(oracle, nodes, counts, conc[1], SAMPLE)
    sess.close()
    ctx.close()
