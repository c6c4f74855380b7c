"""PointCloud2 messages from the push (rpl_capsule_stream_push_cloud_msgs[_dev]) against a push followed by
rpl_capsule_stream_cloud_msgs[_dev]; prints one JSON line.

Shapes (dense capsules, 0x85; every push continues the streams; a pool of 8 pushes is replayed in turn):
  * aggregator: 256 streams x 320 capsules per push (4 revolutions), max_nodes 4096, max_scans 4;
  * live: 512 streams x 80 capsules per push (one revolution), max_nodes 8192, max_scans 2.
Each shape runs three cloud chains: the range / intensity window only, a 5 cm voxel grid, and SOR (k = 8) + 5 cm voxels.
Reported per shape, chain and push, all pushes stamped:
  * host: push_ts (host buffers) + cloud_msgs against push_cloud_msgs, wall time of the synchronous calls;
  * dev: push_ts_dev + cloud_msgs_dev against push_cloud_msgs_dev, CUDA events on one stream;
  * bytes device-to-host of each host form (the push's padded rows and tables, then cloud_msgs' tables and messages;
    against the tables and the messages);
  * device memory of the work blocks, from the layouts (the device push's padded rows the caller provides plus
    cloud_msgs' block of every slot, against the block of one device chunk), and as measured by cudaMemGetInfo around
    each form's first call.
The variants alternate in rounds within one run; each figure is the median over the rounds, with the rounds listed.
The GPU's name and power limit are part of the output.
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

from bench_dense_stream import feed  # noqa: E402
from bench_stream_msgs import gpu_info  # noqa: E402

SHAPES = {"aggregator": (256, 320, 4096, 4), "live": (512, 80, 8192, 2)}
POOL = 8


def chains(R):
    return {"window": R.cloud_params(0.15, 40.0, 0.0),
            "voxel_5cm": R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05),
            "sor8_voxel_5cm": R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)}


def region(b):
    return (b + 255) // 256 * 256


def run_shape(R, torch, n, units, max_nodes, ms, args):
    NS = n * ms
    data = feed(n, units * POOL)  # [n, units * POOL, 84]
    pools = [np.ascontiguousarray(data[:, p * units:(p + 1) * units]) for p in range(POOL)]
    cnt = np.full(n, units, np.uint32)
    prm = R.scan_params(1, 0, 0, 1)
    timing = R.Timing(31, 0, 0, 0)
    rxs = [(10_000_000 + 100_000 * p + np.arange(units, dtype=np.uint64) * 250)[None, :].repeat(n, 0)
           for p in range(POOL)]
    ctx = R.Context(0, max_nodes, NS)
    make = lambda: R.DenseStreamSession(ctx, n, units, max_nodes, ms)  # noqa: E731
    out = {k: R.host_alloc(b).view(dt).reshape(shape) for k, b, dt, shape in (
        ("ranges", NS * max_nodes * 4, np.float32, (NS, max_nodes)),
        ("intensities", NS * max_nodes * 4, np.float32, (NS, max_nodes)),
        ("beam_counts", NS * 4, np.uint32, (NS,)), ("angle_increment", NS * 4, np.float32, (NS,)),
        ("scans_per_stream", n * 4, np.uint32, (n,)), ("scan_begin_ts_us", NS * 8, np.uint64, (NS,)))}
    cap = NS * ((288 + 116 + 16 * max_nodes + 1 + 15) // 16 * 16)
    msgs = R.host_alloc(cap).view(np.uint8)
    msgs2 = R.host_alloc(cap).view(np.uint8)
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
    chunk_dev = min(n, NS // ms)  # the sessions' device chunk (streams), from the context's max_scans
    res = {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms, "chunk_dev": chunk_dev,
           "work_block_bytes": {
               "push_ts_dev_plus_cloud_msgs_dev": NS * max_nodes * 8 + region(NS * max_nodes * 16) + 2 * region(NS * 4),
               "push_cloud_msgs_dev": region(chunk_dev * ms * max_nodes * 16) + region(chunk_dev * ms * 4)}}
    measured = {}
    for name, cp in chains(R).items():
        sa, sb, da, db = make(), make(), make(), make()
        step = [0, 0]
        last = {}

        def run_host(which):
            dt = 0.0
            for _ in range(args.steps):
                p = step[which] % POOL
                step[which] += 1
                t0 = time.perf_counter()
                if which == 0:
                    sa.push(pools[p], cnt, prm, out=out, rx_us=rxs[p], timing=timing)
                    last["a"] = sa.cloud_msgs(cp, 0, msgs=msgs, packed=True)
                else:
                    last["b"] = sb.push_cloud_msgs(pools[p], cnt, cp, 0, rx_us=rxs[p], timing=timing, msgs=msgs2,
                                                   packed=True)[0]
                dt += time.perf_counter() - t0
            return dt / args.steps * 1e3

        k = [0, 0]

        def run_dev(which):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                p = k[which] % POOL
                k[which] += 1
                if which == 0:
                    da.push_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                                inc.data_ptr(), sps.data_ptr(), stream=st.cuda_stream, rx_us=d_rx[p].data_ptr(),
                                timing=timing, scan_begin_ts_us=ts.data_ptr())
                    da.cloud_msgs_dev(cp, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(), d_sz.data_ptr(),
                                      d_tot.data_ptr(), stream=st.cuda_stream)
                else:
                    db.push_cloud_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), cp, 0, d_msgs.data_ptr(), cap,
                                           d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(), sps.data_ptr(),
                                           rx_us=d_rx[p].data_ptr(), timing=timing, stream=st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps

        if not measured:  # each device form's first call allocates its session's blocks
            torch.cuda.synchronize()
            for which, key in ((0, "push_ts_dev_plus_cloud_msgs_dev"), (1, "push_cloud_msgs_dev")):
                f0 = torch.cuda.mem_get_info()[0]
                saved = args.steps
                args.steps = 1
                run_dev(which)
                args.steps = saved
                measured[key] = f0 - torch.cuda.mem_get_info()[0]
        for _ in range(args.warmup):
            run_host(0)
            run_host(1)
            run_dev(0)
            run_dev(1)
        host = {"push_ts_plus_cloud_msgs": [], "push_cloud_msgs": []}
        devt = {"push_ts_dev_plus_cloud_msgs_dev": [], "push_cloud_msgs_dev": []}
        for _ in range(args.rounds):
            host["push_ts_plus_cloud_msgs"].append(run_host(0))
            host["push_cloud_msgs"].append(run_host(1))
            devt["push_ts_dev_plus_cloud_msgs_dev"].append(run_dev(0))
            devt["push_cloud_msgs_dev"].append(run_dev(1))
        a, b = last["a"], last["b"]
        assert a["total_bytes"] == b["total_bytes"] and (a["msg_sizes"] == b["msg_sizes"]).all()
        n_chunks = -(-n // chunk_dev)  # the host chunks are at most the device chunks
        med = lambda v: float(np.median(v))  # noqa: E731
        spread = lambda v: [float(min(v)), float(max(v))]  # noqa: E731
        res[name] = {
            "messages_per_push": int((b["msg_sizes"] > 0).sum()), "message_bytes_per_push": b["total_bytes"],
            "host_ms": {k2: med(v) for k2, v in host.items()}, "dev_ms": {k2: med(v) for k2, v in devt.items()},
            "host_ms_range": {k2: spread(v) for k2, v in host.items()},
            "dev_ms_range": {k2: spread(v) for k2, v in devt.items()},
            "d2h_bytes": {
                "push_ts_plus_cloud_msgs": 2 * NS * max_nodes * 4 + NS * 16 + n * 4 + NS * 12 + 8 + a["total_bytes"],
                "push_cloud_msgs_at_least": NS * 12 + n * 4 + 24 * n_chunks + b["total_bytes"]},
            "rounds": {"host": host, "dev": devt},
        }
        for x in (sa, sb, da, db):
            x.close()
    res["work_block_bytes_measured"] = measured
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
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
