"""The host-buffer calls of a context share one growable device staging block per lane: rpl_scan_batch,
rpl_cloud_batch, rpl_chain_dense_laserscan, the stream sessions' host pushes (stamped or not) and the single-stream
decoders.  One context serving every kind interleaved, with sizes that grow and shrink from call to call (so the
blocks are regrown between calls), returns for each call what the same call returns on a fresh context, bit for bit.
What a call leaves unwritten is not compared: ranges past a scan's beam count, points past a cloud's point count,
scan slots past a stream's published scans."""
import numpy as np
import pytest

from test_capsule_oracle_vs_ref import make_capsules
from test_decode_oracle_vs_ref import make_stream
from test_gpu_capsule_stream import _scans
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS, rx_times

pytestmark = pytest.mark.gpu

CTX_NODES, CTX_SCANS = 8192, 512
MAX_NODES, MAX_SCANS = 4096, 8  # per stream of the chain and the sessions: 64 streams per chunk of the context
NORMAL_SCANS = 48  # a stretch of noise bytes can open many short 0x81 scans
PARAMS = (1, 0, 0, 1)  # is_new_protocol, scan_processing (Mode B), inverted, apply_ascend


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _scan_rows(out, n, max_scans=MAX_SCANS):
    """the published scans of a chain call or a push, with the stamps of a stamped push"""
    rows = [_scans(out, n, max_scans), _bits(out["scans_per_stream"])]
    if "scan_begin_ts_us" in out:
        rows.append(_bits(out["scan_begin_ts_us"]))  # unused slots are written 0
    return rows


def _dense(O, n, n_caps, seed):
    caps = np.stack([make_stream(O, n_caps, 80.0 + s % 5, seed=seed + s, sync_every=150 + s % 7) for s in range(n)])
    counts = np.full(n, n_caps, np.uint32)
    counts[1::5] = n_caps // 3
    return caps, counts


def _scan_batch(R, O, f, seed):
    caps, _ = _dense(O, 1, 300 * f, seed)
    nodes = O.dense_decode(caps[0], 31, 0)[0].view(np.uint8).reshape(-1, 8)
    stride = (1600, 9000, 3200)[f % 3]  # the shared-memory kernels, and above 8192 nodes the large-scan ones
    n_scans = len(nodes) // stride
    buf = np.ascontiguousarray(nodes[: n_scans * stride].reshape(n_scans, stride, 8)).view(R.NODE_DTYPE)[..., 0]
    counts = (min(stride, CTX_NODES) - np.arange(n_scans) * 37 % 1000).astype(np.uint32)

    def run(ctx):
        out = ctx.scan_batch(buf, counts, R.scan_params(*PARAMS), emit_nodes=True)
        m = out["beam_counts"]
        return [_bits(out[k]) for k in ("nodes", "beam_counts", "angle_increment", "status", "path")] + \
            [_bits(out[k][s, : m[s]]) for k in ("ranges", "intensities") for s in range(n_scans)]

    return run


def _cloud_batch(R, O, f, seed):
    caps, _ = _dense(O, 1, 90 * f, seed)
    nodes = O.dense_decode(caps[0], 31, 0)[0].view(np.uint8).reshape(-1, 8)
    stride = 2400
    n_scans = len(nodes) // stride
    buf = np.ascontiguousarray(nodes[: n_scans * stride].reshape(n_scans, stride, 8)).view(R.NODE_DTYPE)[..., 0]
    counts = np.full(n_scans, stride - 100, np.uint32)

    def run(ctx):
        xyzi, pc = ctx.cloud_batch(buf, counts, R.cloud_params(range_min=0.15, range_max=40.0, voxel_size=0.05, sor_k=8))
        return [_bits(pc)] + [_bits(xyzi[s, : pc[s]]) for s in range(n_scans)]

    return run


def _chain(R, O, f, seed):
    n = 24 * f  # two chunks from f = 3 on
    caps, counts = _dense(O, n, 200, seed)

    def run(ctx):
        return _scan_rows(ctx.chain_dense_laserscan(caps, counts, R.scan_params(*PARAMS), MAX_NODES, MAX_SCANS), n)

    return run


def _dense_push(R, O, f, seed, stamped):
    n = 20 * f
    caps, counts = _dense(O, n, 240, seed)
    rx = np.stack([rx_times(240, seed + s) for s in range(n)]) if stamped else None
    timing = R.Timing(*TIMINGS[1]) if stamped else None

    def run(ctx):
        with R.DenseStreamSession(ctx, n, 240, MAX_NODES, MAX_SCANS) as sess:
            out = sess.push(caps, counts, R.scan_params(*PARAMS), sample_duration_us=TIMINGS[1][0] if stamped else 31,
                            rx_us=rx, timing=timing)
        return _scan_rows(out, n)

    return run


def _normal_push(R, O, f, seed, stamped):
    n, stride, chunk_bytes = 8 * f, 5 * 7000, 64  # 10 streams per chunk of the context
    buf = np.full((n, stride), 0xEE, np.uint8)
    counts = np.zeros(n, np.uint32)
    for s in range(n):
        b = normal_stream(7000 - 600 * (s % 4), seed + s, nodes_per_rev=2900, noise=50)[:stride]
        buf[s, : len(b)] = b
        counts[s] = len(b)
    n_chunks = -(-stride // chunk_bytes)
    rx = np.stack([rx_times(n_chunks, seed + s) for s in range(n)]) if stamped else None

    def run(ctx):
        with R.NormalStreamSession(ctx, n, stride, MAX_NODES, NORMAL_SCANS) as sess:
            kw = dict(chunk_bytes=chunk_bytes, chunk_rx_us=rx, timing=R.Timing(*TIMINGS[3])) if stamped else {}
            out = sess.push(buf, counts, R.scan_params(*PARAMS), **kw)
        return _scan_rows(out, n, NORMAL_SCANS)

    return run


def _decode_capsules(R, O, f, seed):
    ans = (0x82, 0x84, 0x85, 0x86)[f % 4]
    per = O.capsule_nodes(ans)
    n_caps = 150 * f
    caps = make_stream(O, n_caps, 80.0, seed=seed) if ans == 0x85 else \
        make_capsules(O, ans, n_caps, 3200.0 / per, seed=seed, sync_every=170)
    rx = rx_times(n_caps, seed)

    def run(ctx):
        nodes, status, offs, state, ts = ctx.decode_capsules(ans, caps, TIMINGS[2][0], timing=R.Timing(*TIMINGS[2]),
                                                             capsule_rx_us=rx)
        return [_bits(nodes), _bits(status), _bits(offs), state, _bits(ts)]

    return run


def _decode_normal(R, O, f, seed):
    b = normal_stream(3000 * f, seed, nodes_per_rev=2900, noise=50)

    def run(ctx):
        return [_bits(ctx.decode_normal(b))]

    return run


def test_interleaved_host_calls_match_fresh_contexts(R, oracle):
    O = oracle
    kinds = [
        ("scan_batch", _scan_batch),
        ("cloud_batch", _cloud_batch),
        ("chain", _chain),
        ("dense_push", lambda R, O, f, seed: _dense_push(R, O, f, seed, False)),
        ("decode_capsules", _decode_capsules),
        ("normal_push_ts", lambda R, O, f, seed: _normal_push(R, O, f, seed, True)),
        ("dense_push_ts", lambda R, O, f, seed: _dense_push(R, O, f, seed, True)),
        ("decode_normal", _decode_normal),
        ("normal_push", lambda R, O, f, seed: _normal_push(R, O, f, seed, False)),
    ]
    shared = R.Context(0, CTX_NODES, CTX_SCANS)
    sizes = [1, 4, 2, 5, 1, 3]  # every kind runs at each size in turn: the blocks grow, shrink back and grow again
    for i, f in enumerate(sizes):
        for j, (name, make) in enumerate(kinds):
            run = make(R, O, f, 1000 * i + 100 * j)
            got = run(shared)
            fresh = R.Context(0, CTX_NODES, CTX_SCANS)
            want = run(fresh)
            fresh.close()
            assert got == want, (name, f)
    shared.close()
