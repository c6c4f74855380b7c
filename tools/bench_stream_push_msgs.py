"""LaserScan messages from the push (rpl_capsule_stream_push_laserscan_msgs[_dev]) against a push followed by
rpl_capsule_stream_laserscan_msgs[_dev]; prints one JSON line.

Shapes (every push continues the streams; a pool of 8 pushes is replayed in turn):
  * aggregator: 256 dense-capsule streams (0x85) x 320 capsules per push (4 revolutions), max_nodes 4096, max_scans 4 --
    the shape of bench_stream_msgs.py;
  * live: 512 dense streams x 80 capsules per push (one revolution), max_nodes 8192, max_scans 2;
  * byte: 256 raw 0x81 byte streams x 16000 bytes per push (one revolution of 3200 records), max_nodes 4096, max_scans 2.
Reported per shape and push, all pushes stamped:
  * host: push_ts (host buffers) + laserscan_msgs against push_laserscan_msgs, wall time of the synchronous calls;
  * dev: push_ts_dev + laserscan_msgs_dev against push_laserscan_msgs_dev, CUDA events on one stream;
  * bytes device-to-host of each host variant (padded rows and tables + packed messages, against tables + the stretch
    of messages), and the total of the bounds against the exact packed size (the bound's slack).
The variants alternate in rounds within one run.  The GPU's name and power limit are part of the output.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed, feed_normal  # noqa: E402
from bench_stream_msgs import gpu_info  # noqa: E402

SHAPES = {"aggregator": ("dense", 256, 320, 4096, 4), "live": ("dense", 512, 80, 8192, 2),
          "byte": ("normal", 256, 16000, 4096, 2)}
POOL = 8
CHUNK = 64  # bytes per receive time of the byte pushes


def run_shape(R, torch, kind, n, units, max_nodes, ms, args):
    NS = n * ms
    if kind == "dense":
        data = feed(n, units * POOL)  # [n, units * POOL, 84]
        per_push = lambda p: np.ascontiguousarray(data[:, p * units:(p + 1) * units])  # noqa: E731
        make = lambda ctx: R.DenseStreamSession(ctx, n, units, max_nodes, ms)  # noqa: E731
        n_rx = units
    else:
        data = feed_normal(n, units * POOL)
        per_push = lambda p: np.ascontiguousarray(data[:, p * units:(p + 1) * units])  # noqa: E731
        make = lambda ctx: R.NormalStreamSession(ctx, n, units, max_nodes, ms)  # noqa: E731
        n_rx = -(-units // CHUNK)
    cnt = np.full(n, units, np.uint32)
    prm = R.scan_params(1, 0, 0, 1)
    timing = R.Timing(31 if kind == "dense" else 500, 0, 0, 0)
    rx = lambda p: (10_000_000 + 100_000 * p + np.arange(n_rx, dtype=np.uint64) * 250)[None, :].repeat(n, 0)  # noqa: E731
    ctx = R.Context(0, max_nodes, NS)
    pools = [per_push(p) for p in range(POOL)]
    rxs = [rx(p) for p in range(POOL)]
    out = {k: R.host_alloc(b).view(dt).reshape(shape) for k, b, dt, shape in (
        ("ranges", NS * max_nodes * 4, np.float32, (NS, max_nodes)),
        ("intensities", NS * max_nodes * 4, np.float32, (NS, max_nodes)),
        ("beam_counts", NS * 4, np.uint32, (NS,)), ("angle_increment", NS * 4, np.float32, (NS,)),
        ("scans_per_stream", n * 4, np.uint32, (n,)), ("scan_begin_ts_us", NS * 8, np.uint64, (NS,)))}
    cap = NS * ((288 + 36 + 8 * max_nodes + 15) // 16 * 16)
    msgs = R.host_alloc(cap).view(np.uint8)
    msgs2 = R.host_alloc(cap).view(np.uint8)
    sa, sb = make(ctx), make(ctx)

    def host_push(sess, p):
        if kind == "dense":
            return sess.push(pools[p], cnt, prm, out=out, rx_us=rxs[p], timing=timing)
        return sess.push(pools[p], cnt, prm, out=out, chunk_bytes=CHUNK, chunk_rx_us=rxs[p], timing=timing)

    def host_push_msgs(sess, p):
        return sess.push_laserscan_msgs(pools[p], cnt, prm, 0, rx_us=rxs[p], timing=timing,
                                        chunk_bytes=None if kind == "dense" else CHUNK, msgs=msgs2, packed=True)

    step = [0, 0]
    last = {}

    def run_host(which):
        dt = 0.0
        for _ in range(args.steps):
            p = step[which] % POOL
            step[which] += 1
            t0 = time.perf_counter()
            if which == 0:
                host_push(sa, p)
                last["a"] = sa.laserscan_msgs(prm, 0, msgs=msgs, packed=True)
            else:
                last["b"] = host_push_msgs(sb, p)
            dt += time.perf_counter() - t0
        return dt / args.steps * 1e3

    for _ in range(args.warmup):
        run_host(0)
        run_host(1)
    host = {"push_ts_plus_laserscan_msgs": [], "push_laserscan_msgs": []}
    for _ in range(args.rounds):
        host["push_ts_plus_laserscan_msgs"].append(run_host(0))
        host["push_laserscan_msgs"].append(run_host(1))
    a, (b, b_sps) = last["a"], last["b"]
    exact = int(sum(((int(x) + 15) // 16) * 16 for x in b["msg_sizes"]))

    # device forms
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    d_pool = [torch.from_numpy(x).to(dev) for x in pools]
    d_rx = [torch.from_numpy(x.view(np.int64)).to(dev) for x in rxs]
    d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
    r = torch.empty((NS, max_nodes), device=dev)
    it = torch.empty((NS, max_nodes), device=dev)
    bc = torch.empty(NS, dtype=torch.int32, device=dev)
    inc = torch.empty(NS, device=dev)
    sps = torch.empty(n, dtype=torch.int32, device=dev)
    ts = torch.empty(NS, dtype=torch.int64, device=dev)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    da, db = make(ctx), make(ctx)
    k = [0, 0]
    cb = None if kind == "dense" else CHUNK

    def run_dev(which):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            p = k[which] % POOL
            k[which] += 1
            if which == 0:
                if kind == "dense":
                    da.push_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                                inc.data_ptr(), sps.data_ptr(), stream=st.cuda_stream, rx_us=d_rx[p].data_ptr(),
                                timing=timing, scan_begin_ts_us=ts.data_ptr())
                else:
                    da.push_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                                inc.data_ptr(), sps.data_ptr(), stream=st.cuda_stream, chunk_bytes=CHUNK,
                                chunk_rx_us=d_rx[p].data_ptr(), timing=timing, scan_begin_ts_us=ts.data_ptr())
                da.laserscan_msgs_dev(prm, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(), d_sz.data_ptr(),
                                      d_tot.data_ptr(), stream=st.cuda_stream)
            else:
                db.push_laserscan_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, 0, d_msgs.data_ptr(), cap,
                                           d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(), sps.data_ptr(),
                                           rx_us=d_rx[p].data_ptr(), timing=timing, chunk_bytes=cb,
                                           stream=st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for _ in range(args.warmup):
        run_dev(0)
        run_dev(1)
    devt = {"push_ts_dev_plus_laserscan_msgs_dev": [], "push_laserscan_msgs_dev": []}
    for _ in range(args.rounds):
        devt["push_ts_dev_plus_laserscan_msgs_dev"].append(run_dev(0))
        devt["push_laserscan_msgs_dev"].append(run_dev(1))
    for x in (sa, sb, da, db):
        x.close()
    ctx.close()
    tables = NS * 12 + 8 + n * 4
    med = lambda v: float(np.median(v))  # noqa: E731
    return {
        "n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms,
        "messages_per_push": int((b["msg_sizes"] > 0).sum()),
        "host_ms": {k2: med(v) for k2, v in host.items()}, "dev_ms": {k2: med(v) for k2, v in devt.items()},
        "d2h_bytes": {"push_ts_plus_laserscan_msgs": 2 * NS * max_nodes * 4 + NS * 16 + n * 4 + a["total_bytes"] + tables,
                      "push_laserscan_msgs": b["total_bytes"] + tables},
        "bound_total_bytes": b["total_bytes"], "exact_packed_bytes": exact,
        "rounds": {"host": host, "dev": devt},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power}
    for s in args.shapes.split(","):
        res[s] = run_shape(R, torch, *SHAPES[s], args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
