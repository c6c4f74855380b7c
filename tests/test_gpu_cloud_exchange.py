"""The fused cloud's pack and exchange layer on one GPU: rpl_cloud_fuse_dev, rpl_cloud_fuse_push_dev with W ranks
simulated by W gather buffers on one device (the push kernel takes raw device pointers, so rank r's push into W
buffers is exactly what it does over NVLink), rpl_exchange_* at world 1 (no NCCL), and multi_gpu.py's
PeerCloudGather / FusedCloudGather at world 1.  tests/test_gpu_multi_push.py covers two real GPUs.

Covered here: cloud_offsets_kernel's carry across its 1024-thread chunks, every header word and every byte around
the slots (guard bytes after the last one), slot overflow, the argument checks, the exchange's double buffering with
a consumer stream and its offsets growing, and a step with no scans, which must publish an empty cloud rather than
leave the one an earlier step wrote."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HEADER = 256        # rpl_peer_gather_bytes: the 256-byte header of uint32 point counts, one word per rank
GUARD = 4096        # bytes after the last slot that nothing may write
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 4096, 16)
    yield c
    c.close()


def clouds(n_scans, stride, seed, max_count=None, zero_share=0.2):
    """Per-scan clouds [n_scans, stride, 4] with ragged counts, some of them 0."""
    rng = np.random.default_rng(seed)
    xyzi = rng.standard_normal((n_scans, stride, 4)).astype(np.float32)
    hi = stride if max_count is None else max_count
    counts = rng.integers(0, hi + 1, n_scans)
    counts[rng.random(n_scans) < zero_share] = 0
    return xyzi, counts.astype(np.uint32)


def concat(xyzi, counts):
    parts = [xyzi[s, : counts[s]] for s in range(len(counts))]
    return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)


def on_device(xyzi, counts):
    """Device copies; a batch of no scans still gets (unread) buffers: the C-ABI takes no null pointers."""
    import torch

    if len(counts) == 0:
        xyzi, counts = np.zeros((1,) + xyzi.shape[1:], np.float32), np.zeros(1, np.uint32)
    return torch.from_numpy(np.ascontiguousarray(xyzi)).cuda(), torch.from_numpy(counts.view(np.int32)).cuda()


def stream_ptr():
    import torch

    return torch.cuda.current_stream().cuda_stream


def dev_bytes(ptr, nbytes):
    """A zero-copy uint8 view of raw device memory."""
    import torch
    from rplidar_ros2_driver_b200.multi_gpu import _DevMem

    return torch.as_tensor(_DevMem(ptr, (nbytes,), "|u1"), device="cuda")


# ---- rpl_cloud_fuse_dev ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_scans", [1, 1023, 1024, 1025, 2500])
def test_fuse_dev(R, ctx, n_scans):
    import torch

    stride = 37
    xyzi, counts = clouds(n_scans, stride, n_scans)
    if n_scans == 1:
        counts[0] = 29
    x, c = on_device(xyzi, counts)
    fused = torch.full((n_scans * stride + 64, 4), float("nan"), device="cuda")
    offs = torch.full((n_scans,), -1, dtype=torch.int32, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    ctx.cloud_fuse_dev(x.data_ptr(), c.data_ptr(), n_scans, stride, fused.data_ptr(), offs.data_ptr(),
                       total.data_ptr(), stream=stream_ptr())
    torch.cuda.synchronize()
    want = concat(xyzi, counts)
    t = int(total.item())
    assert t == int(counts.sum()) == len(want)
    assert (offs.cpu().numpy().view(np.uint32) == np.concatenate([[0], np.cumsum(counts)[:-1]])).all()
    got = fused.cpu().numpy()
    assert (got[:t].view(np.uint32) == want.view(np.uint32)).all()
    assert np.isnan(got[t:]).all()  # nothing written past the cloud


def test_fuse_dev_with_no_scans_writes_a_zero_total(R, ctx):
    import torch

    x, c = on_device(*clouds(4, 8, 1))
    fused = torch.zeros((32, 4), device="cuda")
    offs = torch.full((4,), -1, dtype=torch.int32, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int32, device="cuda")  # 0xFFFFFFFF
    ctx.cloud_fuse_dev(x.data_ptr(), c.data_ptr(), 0, 8, fused.data_ptr(), offs.data_ptr(), total.data_ptr(),
                       stream=stream_ptr())
    torch.cuda.synchronize()
    assert int(total.item()) == 0
    assert (offs.cpu().numpy() == -1).all()


# ---- rpl_cloud_fuse_push_dev, W ranks on one device -----------------------------------------------------------------
class Peers:
    """W gather buffers (rpl_peer_alloc) with guard bytes, filled with a sentinel, and a host model of what each must
    hold."""

    def __init__(self, ctx, world, slot_points):
        self.ctx, self.world, self.slot_points = ctx, world, slot_points
        self.nbytes = HEADER + world * slot_points * 16 + GUARD
        self.ptrs = [ctx.peer_alloc(self.nbytes)[0] for _ in range(world)]
        self.views = [dev_bytes(p, self.nbytes) for p in self.ptrs]
        for v in self.views:
            v.fill_(SENTINEL)
        self.model = np.full(self.nbytes, SENTINEL, np.uint8)

    def push(self, rank, xyzi, counts, stride):
        import torch

        x, c = on_device(xyzi, counts)
        n = len(counts)
        offs = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        total = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        self.ctx.cloud_fuse_push_dev(x.data_ptr(), c.data_ptr(), n, stride, self.ptrs, rank, self.slot_points,
                                     offs.data_ptr(), total.data_ptr(), stream=stream_ptr())
        torch.cuda.synchronize()
        pts = concat(xyzi, counts)
        assert int(total.item()) == len(pts)
        self.model[4 * rank : 4 * rank + 4] = np.array([len(pts)], np.uint32).view(np.uint8)
        kept = pts[: self.slot_points].view(np.uint8).reshape(-1)
        at = HEADER + rank * self.slot_points * 16
        self.model[at : at + kept.size] = kept

    def check(self, what):
        for p, v in enumerate(self.views):
            got = v.cpu().numpy()
            bad = np.flatnonzero(got != self.model)
            assert bad.size == 0, (what, "buffer", p, "first bad byte", int(bad[0]), "of", self.nbytes)

    def close(self):
        for p in self.ptrs:
            self.ctx.peer_free(p)


@pytest.mark.parametrize("world", [1, 2, 5, 16])
def test_push_into_every_rank_buffer(R, ctx, world):
    """Each rank pushes in turn; after every push each buffer must equal the model byte for byte: header words [0, W)
    hold the totals, words [W, 64) and every slot not yet pushed are untouched, slot r holds rank r's cloud.  Rank 0
    and the last rank overflow their slot: the header holds the whole total, the slot its first slot_points points,
    and the next slot (or the guard bytes) nothing more."""
    slot_points, stride = 300, 100
    peers = Peers(ctx, world, slot_points)
    try:
        for rank in range(world):
            overflow = rank in (0, world - 1)
            xyzi, counts = clouds(5, stride, 100 * world + rank, max_count=None if overflow else 60)
            if overflow:
                counts[:] = stride  # 500 points into a 300-point slot
            peers.push(rank, xyzi, counts, stride)
            peers.check(f"after rank {rank}")
    finally:
        peers.close()


def test_push_with_no_scans_publishes_an_empty_cloud(R, ctx):
    world, slot_points, stride = 5, 300, 100
    peers = Peers(ctx, world, slot_points)
    try:
        for rank in range(world):
            peers.push(rank, *clouds(5, stride, rank, max_count=60), stride)
        peers.check("filled")
        for rank in (3, 0):
            peers.push(rank, np.zeros((0, stride, 4), np.float32), np.zeros(0, np.uint32), stride)
            assert all(int(v[4 * rank : 4 * rank + 4].cpu().numpy().view(np.uint32)[0]) == 0 for v in peers.views)
            peers.check(f"rank {rank} pushed no scans")
    finally:
        peers.close()


def test_push_rejects_bad_arguments(R, ctx):
    import torch

    x, c = on_device(*clouds(2, 8, 3))
    offs = torch.zeros(2, dtype=torch.int32, device="cuda")
    total = torch.zeros(1, dtype=torch.int32, device="cuda")
    peers = Peers(ctx, 2, 64)
    L = ctx._L
    try:
        def call(bases, world, rank):
            arr = (C.c_void_p * max(len(bases), 1))(*[C.c_void_p(int(b)) for b in bases])
            return L.rpl_cloud_fuse_push_dev(ctx._h, C.c_void_p(x.data_ptr()), C.c_void_p(c.data_ptr()), 2, 8, arr,
                                             world, rank, 64, C.c_void_p(offs.data_ptr()),
                                             C.c_void_p(total.data_ptr()), None)

        p0, p1 = peers.ptrs
        assert call([], 0, 0) == R.RESULT_INVALID_DATA
        assert call([p0] * 17, 17, 0) == R.RESULT_INVALID_DATA
        assert call([p0, p1], 2, 2) == R.RESULT_INVALID_DATA
        assert call([p0, p1 + 8], 2, 0) == R.RESULT_INVALID_DATA
        assert call([p0 + 4, p1], 2, 1) == R.RESULT_INVALID_DATA
        torch.cuda.synchronize()
        peers.check("rejected calls write nothing")
        assert call([p0, p1], 2, 1) == R.RESULT_OK
    finally:
        torch.cuda.synchronize()
        peers.close()


# ---- rpl_exchange_* at world 1 --------------------------------------------------------------------------------------
def run_exchange(R, ctx, mode, steps, slot_points, stride=4):
    """One allgather per entry of `steps` ((n_scans, counts or None)); the consumer stream waits for each buffer,
    copies the slot and releases it.  Returns [(count, points), ...] and the expected clouds."""
    import torch

    ex = R.Exchange(ctx, None, 1, 0, slot_points)
    consumer = torch.cuda.Stream()
    keep, snaps, want = [], [], []
    try:
        for i, (n, counts) in enumerate(steps):
            xyzi, rnd = clouds(n, stride, 1000 + i, max_count=2, zero_share=0.1)
            counts = rnd if counts is None else counts
            x, c = on_device(xyzi, counts)
            keep.append((x, c))
            idx = ex.allgather(x.data_ptr(), c.data_ptr(), n, stride, mode=mode, stream=stream_ptr())
            assert idx == i & 1
            ex.wait(idx, stream=consumer.cuda_stream)
            pts, cnt = ex.slot(idx, 0)
            with torch.cuda.stream(consumer):
                snaps.append((dev_bytes(cnt, 4).clone(), dev_bytes(pts, slot_points * 16).clone()))
            ex.release(idx, stream=consumer.cuda_stream)
            want.append(concat(xyzi, counts))
        ex.synchronize()
        torch.cuda.synchronize()
        return [(int(a.cpu().numpy().view(np.uint32)[0]), b.cpu().numpy().view(np.float32).reshape(-1, 4))
                for a, b in snaps], want
    finally:
        ex.close()


@pytest.mark.parametrize("mode", ["nccl", "copy"])
def test_exchange_at_world_1(R, ctx, mode):
    slot_points = 6000
    ns = [100, 700, 1500, 2200, 3000, 3000]  # the offsets scratch grows on the way
    steps = [(n, None) for n in ns]
    steps[4] = (3000, np.full(3000, 4, np.uint32))  # 12000 points: overflows the slot
    got, want = run_exchange(R, ctx, R.EXCHANGE_NCCL if mode == "nccl" else R.EXCHANGE_COPY, steps, slot_points)
    for i, ((count, pts), w) in enumerate(zip(got, want)):
        assert count == len(w), (i, count, len(w))
        k = min(count, slot_points)
        assert (pts[:k].view(np.uint32) == w[:k].view(np.uint32)).all(), i
    assert got[4][0] > slot_points


@pytest.mark.parametrize("mode", ["nccl", "copy"])
def test_exchange_step_with_no_scans_reads_empty(R, ctx, mode):
    """Step 2 reuses the buffer step 0 filled; with no scans its count must read 0, not step 0's."""
    steps = [(50, None), (60, None), (0, None), (70, None)]
    got, want = run_exchange(R, ctx, R.EXCHANGE_NCCL if mode == "nccl" else R.EXCHANGE_COPY, steps, 1000)
    assert got[0][0] > 0
    assert [g[0] for g in got] == [len(w) for w in want] and got[2][0] == 0


# ---- multi_gpu.py at world 1 ----------------------------------------------------------------------------------------
def test_cloud_gathers_at_world_1_equal_fuse_dev(R, ctx):
    import torch
    import torch.distributed as dist
    from rplidar_ros2_driver_b200.multi_gpu import FusedCloudGather, PeerCloudGather

    assert not dist.is_initialized()
    dev = torch.device("cuda")
    n_scans, stride, capacity = 40, 64, 40 * 64
    peer = PeerCloudGather(ctx, capacity, dev)
    fcg = FusedCloudGather(capacity, dev)
    try:
        assert peer.world == 1 and fcg.world == 1
        for step in range(3):
            xyzi, counts = clouds(n_scans, stride, 50 + step)
            x, c = on_device(xyzi, counts)
            fused = torch.full((capacity, 4), float("nan"), device=dev)
            offs = torch.zeros(n_scans, dtype=torch.int32, device=dev)
            total = torch.zeros(1, dtype=torch.int32, device=dev)
            ctx.cloud_fuse_dev(x.data_ptr(), c.data_ptr(), n_scans, stride, fused.data_ptr(), offs.data_ptr(),
                               total.data_ptr(), stream=stream_ptr())
            t = int(total.item())
            assert t == int(counts.sum())
            ref = fused[:t].cpu().numpy()

            offs2 = torch.zeros(n_scans, dtype=torch.int32, device=dev)
            total2 = torch.zeros(1, dtype=torch.int32, device=dev)
            half = peer.push(x.data_ptr(), c.data_ptr(), n_scans, stride, offs2.data_ptr(), total2.data_ptr(),
                             stream=stream_ptr())
            torch.cuda.synchronize()
            assert half == step & 1
            assert int(peer.counts(half)[0].item()) == t == int(total2.item())
            assert (peer.gathered(half)[0, :t].cpu().numpy().view(np.uint32) == ref.view(np.uint32)).all()

            gathered, cnt = fcg(fused, total)
            torch.cuda.synchronize()
            assert int(cnt[0].item()) == t
            assert (gathered[0, :t].cpu().numpy().view(np.uint32) == ref.view(np.uint32)).all()
            assert (fcg.compact().cpu().numpy().view(np.uint32) == ref.view(np.uint32)).all()
    finally:
        torch.cuda.synchronize()
        peer.close()
