"""The edges of a LaserScan Mode B call on the two-CTA cluster kernel (scan_tma.cu, scan_tma_cluster_kernel): the
hand-off counter each call finds zeroed by the previous call's general kernel instead of by a memset of its own, the
general kernel launched as the cluster kernel's programmatic dependent, the self-timed profiling of both, and the
scans the clusters draw at run time from the call's ticket, at every kind of batch size.

Every call is compared bit for bit with the same batch under RPL_FLAG_FORCE_GENERAL (the general kernel alone), and
its `path` with the scans that carry a duplicated measured key: those, and only those, go to the general kernel.  A
count left over from an earlier call would send tie-free scans there too, or (a zero missing) hand on stale scans."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STRIDE = 32768
FORCE_GENERAL = 1
PARAMS = (0, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


def make_batch(R, torch, ctx, seed, n_scans, dups):
    """n_scans synthetic full-length scans on the device; the scans in `dups` get a duplicated measured key (node 5
    and the last node share node 5's angle, both measured)."""
    nodes = torch.empty((n_scans, STRIDE, 8), dtype=torch.uint8, device="cuda")
    counts = torch.empty(n_scans, dtype=torch.int32, device="cuda")
    ctx.synth_batch_dev(seed, n_scans, STRIDE, STRIDE, seed % 2, nodes.data_ptr(), counts.data_ptr())
    torch.cuda.synchronize()
    dist = torch.from_numpy(np.array([4000, 8000], "<u4").view(np.uint8).reshape(2, 4)).cuda()
    for s in dups:
        nodes[s, STRIDE - 1, 0:2] = nodes[s, 5, 0:2]
        nodes[s, 5, 2:6] = dist[0]
        nodes[s, STRIDE - 1, 2:6] = dist[1]
    expect = np.zeros(n_scans, np.uint32)
    expect[list(dups)] = 1
    torch.cuda.synchronize()  # the library's streams do not wait for torch's
    return nodes, counts, expect


class Call:
    """one rpl_scan_batch_dev call's outputs (fresh buffers); issue() enqueues it, host() fetches them"""

    def __init__(self, R, torch, ctx, batch, flags=0):
        self.R, self.ctx, self.flags = R, ctx, flags
        self.nodes, self.counts, self.expect = batch
        S = self.nodes.shape[0]
        self.ranges = torch.full((S, STRIDE), float("nan"), device="cuda")
        self.intens = torch.full((S, STRIDE), float("nan"), device="cuda")
        self.small = [torch.full((S,), 0x7777, dtype=torch.int32, device="cuda") for _ in range(4)]
        torch.cuda.synchronize()  # the fills are done before a library stream writes these buffers

    def issue(self, stream=None):
        S = self.nodes.shape[0]
        self.ctx.scan_batch_dev(self.nodes.data_ptr(), self.counts.data_ptr(), S, STRIDE,
                                self.R.scan_params(*PARAMS, self.flags), ranges=self.ranges.data_ptr(),
                                intensities=self.intens.data_ptr(), beam_counts=self.small[0].data_ptr(),
                                angle_increment=self.small[1].data_ptr(), status=self.small[2].data_ptr(),
                                path=self.small[3].data_ptr(), stream=stream)
        return self

    def host(self):
        b, inc, st, path = (t.cpu().numpy() for t in self.small)
        return {"ranges": self.ranges.cpu().numpy(), "intens": self.intens.cpu().numpy(), "beams": b,
                "inc": inc, "status": st, "path": path.view(np.uint32)}


def reference(R, torch, ctx, batch):
    got = Call(R, torch, ctx, batch, FORCE_GENERAL).issue()
    torch.cuda.synchronize()
    return got.host()


def check(got, ref, expect, tag):
    assert (got["path"] == expect).all(), (tag, np.nonzero(got["path"] != expect)[0][:8])
    for k in ("beams", "inc", "status"):
        assert (got[k] == ref[k]).all(), (tag, k)
    for s in range(len(expect)):
        m = int(ref["beams"][s])
        for k in ("ranges", "intens"):
            assert (got[k][s, :m].view(np.uint32) == ref[k][s, :m].view(np.uint32)).all(), (tag, k, s)


# 140 scans: more than two rounds of the 66 clusters of an H100, so every cluster meets several scans
N_SCANS = 140
DUPS = (3, 70, 71, 139)


def batches(R, torch, ctx):
    dup = make_batch(R, torch, ctx, 101, N_SCANS, DUPS)
    clean = make_batch(R, torch, ctx, 202, N_SCANS, ())
    return [(b, reference(R, torch, ctx, b)) for b in (dup, clean)]


def test_alternating_calls_on_one_lane(R, torch):
    ctx = R.Context(0, STRIDE, N_SCANS)
    pairs = batches(R, torch, ctx)
    for i in range(6):  # handed-on, tie-free, handed-on, ...; every call on the context's own stream
        batch, ref = pairs[i % 2]
        got = Call(R, torch, ctx, batch).issue()
        ctx.synchronize()
        check(got.host(), ref, batch[2], i)


def test_alternating_calls_on_two_streams(R, torch):
    ctx = R.Context(0, STRIDE, N_SCANS)
    pairs = batches(R, torch, ctx)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    calls = [Call(R, torch, ctx, pairs[i % 2][0]).issue(streams[(i // 2) % 2].cuda_stream) for i in range(8)]
    torch.cuda.synchronize()
    for i, c in enumerate(calls):
        check(c.host(), pairs[i % 2][1], pairs[i % 2][0][2], i)


def test_failed_call_then_good_call(R, torch):
    ctx = R.Context(0, STRIDE, N_SCANS)
    pairs = batches(R, torch, ctx)
    (dup, ref_dup), (clean, ref_clean) = pairs
    Call(R, torch, ctx, dup).issue()  # leaves hand-offs in this call's counter
    bad = Call(R, torch, ctx, clean)
    with pytest.raises(R.RplError):  # ranges without intensities: refused before any launch
        ctx.scan_batch_dev(bad.nodes.data_ptr(), bad.counts.data_ptr(), N_SCANS, STRIDE, R.scan_params(*PARAMS),
                           ranges=bad.ranges.data_ptr())
    with pytest.raises(R.RplError):  # more scans than the context holds
        ctx.scan_batch_dev(bad.nodes.data_ptr(), bad.counts.data_ptr(), N_SCANS + 1, STRIDE, R.scan_params(*PARAMS),
                           ranges=bad.ranges.data_ptr(), intensities=bad.intens.data_ptr())
    for batch, ref in ((clean, ref_clean), (dup, ref_dup), (clean, ref_clean)):
        got = Call(R, torch, ctx, batch).issue()
        ctx.synchronize()
        check(got.host(), ref, batch[2], "after a refused call")


def test_cloud_post_passes_after_cluster_calls(R, oracle, torch):
    """rpl_cloud_batch_dev's post passes read the hand-off list and count after the general kernel, restricted to the
    scans the fused kernel handed on: after Mode B cluster calls that handed scans on (and one that did not), they
    must give what they give on a fresh context."""
    n, S = 3200, 24
    nodes = oracle.synth_batch(300, S, n, 4)
    for s in (2, 9, 17):  # duplicated measured keys: handed to the general kernel, then to the restricted passes
        nodes["angle_z_q14"][s, n - 1] = nodes["angle_z_q14"][s, 7]
        nodes["dist_mm_q2"][s, [7, n - 1]] = [4000, 8000]
    counts = np.full(S, n, np.uint32)
    prm = R.cloud_params(range_min=0.15, range_max=40.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)
    d_nodes = torch.from_numpy(nodes.view(np.uint8).reshape(S, n * 8)).cuda()
    d_counts = torch.from_numpy(counts.view(np.int32)).cuda()
    torch.cuda.synchronize()

    def cloud(ctx):
        xyzi = torch.full((S, n, 4), float("nan"), device="cuda")
        pc = torch.zeros(S, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.cloud_batch_dev(d_nodes.data_ptr(), d_counts.data_ptr(), S, n, prm, xyzi.data_ptr(), pc.data_ptr())
        ctx.synchronize()
        pc = pc.cpu().numpy()
        x = xyzi.cpu().numpy()
        return pc, [x[s, :pc[s]].copy() for s in range(S)]

    fresh = R.Context(0, STRIDE, N_SCANS)
    want_pc, want = cloud(fresh)
    ctx = R.Context(0, STRIDE, N_SCANS)
    (dup, ref_dup), (clean, _) = batches(R, torch, ctx)
    for lead in (dup, clean, dup):
        Call(R, torch, ctx, lead).issue()
        pc, got = cloud(ctx)
        assert (pc == want_pc).all()
        for s in range(S):
            assert (got[s].view(np.uint32) == want[s].view(np.uint32)).all(), s
    got = Call(R, torch, ctx, dup).issue()  # and a cluster call after the cloud call
    ctx.synchronize()
    check(got.host(), ref_dup, dup[2], "after a cloud call")


def test_session_clouds_between_cluster_calls(R, oracle, torch):
    """A stream session's pushes and cloud calls (the chunk driver reads the hand-off list and count after the general
    kernel: HQ revolutions with duplicate measured keys, some longer than the fused kernel's 4096 nodes) with Mode B
    cluster calls that hand scans on before and after each of them: the same scans and clouds as with none."""
    from test_gpu_capsule_stream import _scans
    from test_gpu_stream_cloud import MAX_SCANS, REV_NODES, SETTINGS, Feed, cloud_rows, hq_stream, prm_of, splits

    feed = Feed(R, oracle, "framed", 0x83)
    n = 8
    streams = [hq_stream(oracle, 4, REV_NODES[s % 4] + s // 4, 700 + s, dup_share=0.002 if s % 3 else 0.0)
               for s in range(n)]
    pieces = splits(np.random.default_rng(8192), streams, 2)
    stride = max(len(p) for push in pieces for p in push)
    settings = [prm_of(R, f, **kw) for kw in SETTINGS[1:] for f in (0, R.CLOUD_NO_FUSED)]

    def session_run(ctx, lead):
        out_rows = []
        with feed.session(ctx, n, stride, 8192) as sess:
            for push in pieces:
                lead()
                out = feed.push(sess, push, stride)
                out_rows.append(_scans(out, n, MAX_SCANS))
                for prm in settings:
                    lead()
                    out_rows.append(cloud_rows(sess.cloud(prm), out["scans_per_stream"], n, MAX_SCANS))
        return out_rows

    want = session_run(R.Context(0, STRIDE, N_SCANS), lambda: None)
    ctx = R.Context(0, STRIDE, N_SCANS)
    (dup, ref_dup), _ = batches(R, torch, ctx)
    leads = []

    def lead():
        leads.append(Call(R, torch, ctx, dup).issue())

    assert session_run(ctx, lead) == want
    ctx.synchronize()
    for i, c in enumerate(leads):
        check(c.host(), ref_dup, dup[2], ("lead", i))


def test_profiling_keeps_outputs_and_counts_launches(R, torch):
    ctx = R.Context(0, STRIDE, N_SCANS)
    (dup, ref_dup), (clean, ref_clean) = batches(R, torch, ctx)
    ctx.profile_read()
    ctx.profile(True)
    calls = [Call(R, torch, ctx, b).issue() for b in (dup, clean, dup, clean, dup)]
    fast_ms, fast_n, general_ms, general_n = ctx.profile_read()
    ctx.profile(False)
    assert (fast_n, general_n) == (5, 5)
    assert fast_ms > 0 and general_ms > 0
    for i, c in enumerate(calls):
        check(c.host(), *((ref_dup, dup[2]) if i % 2 == 0 else (ref_clean, clean[2])), i)
    assert ctx.profile_read()[1::2] == (0, 0)  # nothing profiled since the last read
    got = Call(R, torch, ctx, dup).issue()  # profiling off again
    ctx.synchronize()
    check(got.host(), ref_dup, dup[2], "profiling off")


@pytest.mark.parametrize("n_scans", [1, 65, 66, 67, 4096])
def test_cluster_batch_sizes(R, torch, n_scans):
    """fewer scans than clusters, one round exactly, one scan over, and the headline batch"""
    ctx = R.Context(0, STRIDE, n_scans)
    dups = sorted({0, n_scans // 2, n_scans - 1})
    batch = make_batch(R, torch, ctx, 7 + n_scans, n_scans, dups if n_scans > 1 else ())
    ref = reference(R, torch, ctx, batch)
    for _ in range(2):
        got = Call(R, torch, ctx, batch).issue()
        ctx.synchronize()
        check(got.host(), ref, batch[2], n_scans)


@pytest.mark.parametrize("n_scans", [67, 140, 4096])
def test_scans_left_out_of_the_sequence(R, torch, n_scans):
    """empty scans and scans longer than the stride, among the clusters' first two scans and among the ones drawn at
    run time: reported by the cluster kernel (path 0) as the general kernel reports them, the others unchanged"""
    ctx = R.Context(0, STRIDE, n_scans)
    nodes, counts, expect = make_batch(R, torch, ctx, 31 + n_scans, n_scans, [n_scans // 3])
    rng = np.random.default_rng(n_scans)
    odd = sorted(set(rng.choice(n_scans, min(n_scans // 4, 200), replace=False).tolist()) | {0, n_scans - 1} -
                 {n_scans // 3})
    for i, s in enumerate(odd):
        counts[s] = 0 if i % 2 else STRIDE + 1
    expect[odd] = 0
    torch.cuda.synchronize()
    batch = (nodes, counts, expect)
    ref = reference(R, torch, ctx, batch)
    for _ in range(2):
        got = Call(R, torch, ctx, batch).issue()
        ctx.synchronize()
        check(got.host(), ref, expect, n_scans)
