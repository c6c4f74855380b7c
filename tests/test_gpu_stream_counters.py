"""rpl_capsule_stream_counters (CapsuleStreamSession.counters): the counters the stream sessions accumulate on the device,
held after the last push exactly to the restatement of the whole stream (tests/test_stream_counters_pieces.py, pinned
against the SDK there), for framed sessions of 0x82..0x86 and byte sessions of 0x81..0x86, damaged streams split into
seeded random pushes (zero-length ones included) through every push flavour mixed on one session.  scans_unreturned is
held to what the pushes returned, bytes_in of a byte session to the byte identity with state()'s held bytes."""
import numpy as np
import pytest

from test_capsule_stream_pieces import format_stream
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_stream_counters_pieces import FIELDS, frame_size, golden_stream, restated_counters

pytestmark = pytest.mark.gpu

MAX_NODES, MAX_SCANS = 1024, 1
FLAVOURS = ("host", "dev", "host_ts", "dev_ts")
PARAMS = (1, 0, 0, 1)
# what one push of each flavour launches on a 4-stream session (capsule_stream_chunk: framer, decoder, assembler, scan
# kernels), taken from the build before the counters: counting adds no launch
# (measured on the parent: 0x81 bytes 4 = decoder, assembler, two scan launches; capsule bytes 5 = framer + those 4;
# framed 4)
PARENT_LAUNCHES = {f"{k}-{a:02x}-{f}": n for k, a, n in [("bytes", 0x81, 4)] + [("bytes", a, 5) for a in range(0x82, 0x87)]
                   + [("framed", a, 4) for a in range(0x82, 0x87)] for f in ("host", "dev", "host_ts", "dev_ts")}


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


class Sess:
    """a session of either kind and its pushes in any flavour; `unreturned` sums max(0, scans_per_stream - max_scans)"""

    def __init__(self, R, ctx, ans, byte, n, stride, max_scans=MAX_SCANS):
        self.R, self.ans, self.byte, self.n, self.stride, self.max_scans = R, ans, byte, n, stride, max_scans
        self.cb = 1 if ans == 0x81 else R.lib().rpl_capsule_bytes(ans)
        if byte:
            self.sess = R.CapsuleByteStreamSession(ctx, ans, n, stride, MAX_NODES, max_scans)
        else:
            self.sess = R.CapsuleStreamSession(ctx, ans, n, stride, MAX_NODES, max_scans)
        self.unreturned = np.zeros(n, np.int64)
        self.chunk_bytes = 3 * self.cb + 1

    def _buf(self, push):
        shape = (self.n, self.stride) if self.byte else (self.n, self.stride, self.cb)
        buf = np.full(shape, 0xEE, np.uint8)
        cnt = np.zeros(self.n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        return buf, cnt

    def _rx(self, t):
        cols = -(-self.stride // self.chunk_bytes) if self.byte else self.stride
        return (1_000_000 * (t + 1) + np.arange(self.n * cols, dtype=np.uint64)).reshape(self.n, cols)

    def push(self, push, flavour, t, params=None, timing=None):
        R = self.R
        params = params or R.scan_params(*PARAMS)
        timing = timing or R.Timing(31, 0, 0, 0)
        buf, cnt = self._buf(push)
        ts = flavour.endswith("_ts")
        if flavour.startswith("host"):
            if not ts:
                out = self.sess.push(buf, cnt, params)
            elif self.byte:
                out = self.sess.push(buf, cnt, params, chunk_bytes=self.chunk_bytes, chunk_rx_us=self._rx(t),
                                     timing=timing)
            else:
                out = self.sess.push(buf, cnt, params, rx_us=self._rx(t), timing=timing)
            sps = out["scans_per_stream"]
        else:
            sps = self._push_dev(buf, cnt, params, ts, t, timing)
        self.unreturned += np.maximum(sps.astype(np.int64) - self.max_scans, 0)
        return sps

    def _push_dev(self, buf, cnt, params, ts, t, timing, stream=None):
        import torch

        dev = torch.device("cuda", 0)
        NS = self.n * self.max_scans
        d_buf = torch.from_numpy(buf).to(dev)
        d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
        r = torch.zeros((NS, MAX_NODES), device=dev)
        it = torch.zeros((NS, MAX_NODES), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, dtype=torch.float32, device=dev)
        sps = torch.zeros(self.n, dtype=torch.int32, device=dev)
        d_ts = torch.zeros(NS, dtype=torch.int64, device=dev)
        d_rx = torch.from_numpy(self._rx(t).view(np.int64)).to(dev)
        torch.cuda.synchronize()
        args = (d_buf.data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(), bc.data_ptr(), inc.data_ptr(),
                sps.data_ptr())
        kw = dict(stream=stream)
        if ts and self.byte:
            kw.update(chunk_bytes=self.chunk_bytes, chunk_rx_us=d_rx.data_ptr(), timing=timing,
                      scan_begin_ts_us=d_ts.data_ptr())
        elif ts:
            kw.update(rx_us=d_rx.data_ptr(), timing=timing, scan_begin_ts_us=d_ts.data_ptr())
        self.sess.push_dev(*args, **kw)
        self.sess._ctx.synchronize()
        return sps.cpu().numpy().view(np.uint32)

    def close(self):
        self.sess.close()


def _streams(O, ans, byte, n, seed):
    if byte:
        return [golden_stream(O, ans, seed + s) for s in range(n)]
    return [format_stream(O, ans, 150 if ans == 0x83 else 500, seed + s, sync_every=100 + 7 * s) for s in range(n)]


def _split(O, ans, byte, streams, rng):
    fs = frame_size(O, ans) if byte else 1
    sizes = [0, 1, 2, fs - 1, fs, fs + 1, 3 * fs + 7, 40 * fs] if byte else [0, 1, 2, 7, 40, 161]
    # and pieces of half and all the stream, which publish more scans than max_scans returns
    cuts = [_random_cuts(rng, len(b), sizes + [len(b) // 2, len(b)]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    assert any(len(p) == 0 for push in pieces[:-1] for p in push)
    return pieces, max(1, max(len(p) for push in pieces for p in push))


def _check(O, got, streams, ans, byte, sess, sd=31):
    for s, b in enumerate(streams):
        exp, _, held = restated_counters(O, ans, b, MAX_NODES, byte, sd)
        exp["scans_unreturned"] = int(sess.unreturned[s])
        row = {k: int(got[k][s]) for k in FIELDS}
        assert row == exp, (hex(ans), byte, s, {k: (row[k], exp[k]) for k in FIELDS if row[k] != exp[k]})
    if byte:
        state = sess.sess.state()
        held = state[-1]
        fs = frame_size(O, ans)
        assert (got["bytes_in"] == got["frames"] * fs + got["skipped_bytes"] + held).all()


KINDS = [(a, True) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)] + [(a, False) for a in (0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("ans,byte", KINDS, ids=[f"{'bytes' if b else 'framed'}-{a:02x}" for a, b in KINDS])
def test_counters_are_the_restated_whole_streams(R, oracle, ans, byte):
    O = oracle
    n = 4
    rng = np.random.default_rng(ans + 7 * byte)
    streams = _streams(O, ans, byte, n, 71)
    pieces, stride = _split(O, ans, byte, streams, rng)
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    sess = Sess(R, ctx, ans, byte, n, stride)
    got = sess.sess.counters()
    assert all((got[k] == 0).all() for k in FIELDS)
    for t, push in enumerate(pieces):
        sess.push(push, FLAVOURS[int(rng.integers(0, 4))], t)
    got = sess.sess.counters()
    _check(O, got, streams, ans, byte, sess)
    assert (got["scans_unreturned"] > 0).any() and (ans == 0x81 or (got["checksum_errors"] > 0).any())
    assert not byte or (got["nodes_overwritten"] > 0).any()
    assert byte == (got["skipped_bytes"] > 0).any()
    # a second read changes nothing; clear zeroes only the masked streams, which then count from zero again
    again = sess.sess.counters(clear=[1, 0, 1, 0])
    assert (again == got).all()
    after = sess.sess.counters()
    assert (after[[1, 3]] == got[[1, 3]]).all() and all((after[k][[0, 2]] == 0).all() for k in FIELDS)
    sess.close()
    ctx.close()


@pytest.mark.parametrize("ans", [0x85, 0x86])
def test_per_stream_sample_durations_discard_differently(R, oracle, ans):
    """RPL_FLAG_PER_STREAM: two streams of the same capsules, each counted under its own sample duration"""
    O = oracle
    caps = format_stream(O, ans, 400, 77, sync_every=120)
    base = O.decode_capsules(ans, caps, 31)[1] & O.CAPSULE_DISCARD
    sd = next(d for d in (20, 15, 10, 5, 2, 1) if ((O.decode_capsules(ans, caps, d)[1] & O.CAPSULE_DISCARD) != base).any())
    rng = np.random.default_rng(ans)
    pieces, stride = _split(O, ans, False, [caps, caps], rng)
    ctx = R.Context(0, MAX_NODES, 2 * MAX_SCANS)
    sess = Sess(R, ctx, ans, False, 2, stride)
    sess.sess.set_lidars([R.lidar_settings(1, 0, 0, R.Timing(31, 0, 0, 0)), R.lidar_settings(1, 0, 0, R.Timing(sd, 0, 0, 0))])
    params = R.scan_params(*PARAMS, R.FLAG_PER_STREAM)
    for t, push in enumerate(pieces):
        sess.push(push, FLAVOURS[t % 4], t, params=params)
    got = sess.sess.counters()
    for s, d in enumerate((31, sd)):
        exp, _, _ = restated_counters(O, ans, caps, MAX_NODES, False, d)
        exp["scans_unreturned"] = int(sess.unreturned[s])
        assert {k: int(got[k][s]) for k in FIELDS} == exp, (s, d)
    assert got["discarded_capsules"][0] != got["discarded_capsules"][1]
    sess.close()
    ctx.close()


def test_reset_leaves_counters_and_identity_holds_after(R, oracle):
    """a reset drops the held bytes uncounted and leaves the counters; the identity then holds from the reset on"""
    O = oracle
    ans, n = 0x84, 2
    streams = _streams(O, ans, True, n, 90)
    cut = [len(b) // 2 + 5 for b in streams]  # inside a frame
    stride = max(len(b) for b in streams)
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    sess = Sess(R, ctx, ans, True, n, stride)
    sess.push([b[:c] for b, c in zip(streams, cut)], "host", 0)
    before = sess.sess.counters()
    held = sess.sess.state()[2].astype(np.int64)
    sess.sess.reset()
    assert (sess.sess.counters() == before).all()
    sess.push([b[c:] for b, c in zip(streams, cut)], "dev", 1)
    got = sess.sess.counters()
    held_end = sess.sess.state()[2]
    fs = frame_size(O, ans)
    lhs = got["bytes_in"].astype(np.int64) - held
    assert (lhs == got["frames"] * fs + got["skipped_bytes"] + held_end).all()
    sess.close()
    ctx.close()


def test_two_streams_and_null_session(R, oracle):
    """push_dev on two CUDA streams, then counters(): both pushes are seen; a null session is refused"""
    import torch

    O = oracle
    ans, n = 0x85, 2
    caps = [format_stream(O, ans, 300, 5 + s, sync_every=110) for s in range(n)]
    ctx = R.Context(0, MAX_NODES, n * MAX_SCANS)
    sess = Sess(R, ctx, ans, False, n, 300)
    dev = torch.device("cuda", 0)
    NS = n * MAX_SCANS
    keep = []
    for t, st in enumerate((torch.cuda.Stream(), torch.cuda.Stream())):
        buf, cnt = sess._buf([c[150 * t: 150 * (t + 1)] for c in caps])
        bufs = [torch.from_numpy(buf).to(dev), torch.from_numpy(cnt.view(np.int32)).to(dev),
                torch.zeros((NS, MAX_NODES), device=dev), torch.zeros((NS, MAX_NODES), device=dev),
                torch.zeros(NS, dtype=torch.int32, device=dev), torch.zeros(NS, device=dev),
                torch.zeros(n, dtype=torch.int32, device=dev)]
        torch.cuda.synchronize()
        keep.append(bufs)
        ptrs = [b.data_ptr() for b in bufs]
        sess.sess.push_dev(ptrs[0], ptrs[1], R.scan_params(*PARAMS), *ptrs[2:], stream=st.cuda_stream)
    got = sess.sess.counters()
    for s in range(n):
        exp, _, _ = restated_counters(O, ans, caps[s], MAX_NODES, False)
        assert int(got["frames"][s]) == 300 and int(got["nodes"][s]) == exp["nodes"]
    torch.cuda.synchronize()
    L = R.lib()
    assert L.rpl_capsule_stream_counters(None, None, None) == R.capi.RESULT_INVALID_DATA
    sess.close()
    ctx.close()


def launch_deltas(R, O):
    """launches of one push of each flavour on 4-stream sessions of every kind (the parent's are PARENT_LAUNCHES)"""
    out = {}
    for ans, byte in KINDS:
        streams = _streams(O, ans, byte, 4, 31)
        piece = [b[: len(b) // 3] for b in streams]
        stride = max(len(p) for p in piece)
        ctx = R.Context(0, MAX_NODES, 4 * MAX_SCANS)
        sess = Sess(R, ctx, ans, byte, 4, stride)
        for t, f in enumerate(FLAVOURS):
            c0 = ctx.launch_count
            sess.push(piece, f, t)
            out[f"{'bytes' if byte else 'framed'}-{ans:02x}-{f}"] = ctx.launch_count - c0
        sess.close()
        ctx.close()
    return out


def test_launches_per_push_are_the_parents(R, oracle):
    assert launch_deltas(R, oracle) == PARENT_LAUNCHES
