"""LaserScans and their projected clouds from the push (rpl_capsule_stream_push_scan_cloud_msgs[_dev]) against the two
calls it replaces, on the dense shapes of bench_stream_scan_filters.py (DESIGN.md 5.7.1); prints one JSON line.

Every shape has three sessions, each continuing its own streams through a pool of POOL stamped dense pushes (0x85,
Mode B) replayed in turn:
  * floor: push_laserscan_msgs alone;
  * two_calls: push_laserscan_msgs, then scan_cloud_msgs, which replays the push's scan kernels and filters;
  * push_scan_cloud: push_scan_cloud_msgs, which projects the push's own LaserScan messages.
Each runs with laser_geometry's default channels (intensity, index), without and with RPL_FLAG_PER_STREAM_FILTERS
(every stream the whole filter chain and a footprint box).  The device forms are timed with CUDA events on one CUDA
stream, the host forms by wall time of the synchronous calls, with the bytes each moves device-to-host.  The variants
alternate in rounds within one run; each figure is the median over the rounds, with the rounds listed.  The GPU's
name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed  # noqa: E402
from bench_stream_scan_filters import POOL, SHAPES, gpu_info  # noqa: E402

VARIANTS = ("floor", "two_calls", "push_scan_cloud")


def run_shape(R, torch, n, units, max_nodes, ms, args):
    NS = n * ms
    data = feed(n, units * POOL)
    pools = [np.ascontiguousarray(data[:, p * units:(p + 1) * units]) for p in range(POOL)]
    rxs = [(10_000_000 + 100_000 * p + np.arange(units, dtype=np.uint64) * 250)[None, :].repeat(n, 0)
           for p in range(POOL)]
    cnt = np.full(n, units, np.uint32)
    timing = R.Timing(31, 0, 0, 0)
    cp = R.scan_cloud_params()
    ctx = R.Context(0, max_nodes, NS)
    scap = NS * ((288 + 32 + 8 * max_nodes + 4 + 15) // 16 * 16)
    ccap = NS * ((288 + 192 + 20 * max_nodes + 1 + 15) // 16 * 16)
    filt = [R.scan_filter_settings(mask=[(2.8, 3.4)], range_lo=0.15, range_hi=12.0, intensity_min=1.0,
                                   speckle_window=3, speckle_min_neighbours=2, speckle_max_diff=0.05, shadow_window=8,
                                   shadow_angle=math.radians(10))] * n
    box = [R.scan_footprint([[(-0.4, -0.3), (0.4, -0.3), (0.4, 0.3), (-0.4, 0.3)]])] * n

    def session():
        s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
        s.set_frames([f"laser_{k}" for k in range(n)])
        s.set_scan_filters(filt)
        s.set_scan_footprints(box)
        return s

    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    d_pool = [torch.from_numpy(x).to(dev) for x in pools]
    d_rx = [torch.from_numpy(x.view(np.int64)).to(dev) for x in rxs]
    d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    d_sets = []
    for cap in (scap, ccap):
        t = dict(msgs=torch.empty(cap, dtype=torch.uint8, device=dev), offs=torch.empty(NS, dtype=torch.int64, device=dev),
                 sizes=torch.empty(NS, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        t["out"] = R.MsgsOut(t["msgs"].data_ptr(), cap, t["offs"].data_ptr(), t["sizes"].data_ptr(),
                             t["total"].data_ptr())
        d_sets.append(t)
    h_msgs = [R.host_alloc(scap).view(np.uint8), R.host_alloc(ccap).view(np.uint8)]

    res = {}
    for filtered in (False, True):
        prm = R.scan_params(0, 0, 0, 1, R.FLAG_PER_STREAM_FILTERS if filtered else 0)
        sess = {k: session() for k in VARIANTS}
        step = {k: 0 for k in VARIANTS}
        S, C = d_sets

        def dev_call(k, p):
            s = sess[k]
            if k == "push_scan_cloud":
                s.push_scan_cloud_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, cp, 0, S["out"], C["out"],
                                           d_sps.data_ptr(), rx_us=d_rx[p].data_ptr(), timing=timing,
                                           stream=st.cuda_stream)
                return
            s.push_laserscan_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, 0, S["msgs"].data_ptr(), scap,
                                      S["offs"].data_ptr(), S["sizes"].data_ptr(), S["total"].data_ptr(),
                                      d_sps.data_ptr(), rx_us=d_rx[p].data_ptr(), timing=timing, stream=st.cuda_stream)
            if k == "two_calls":
                s.scan_cloud_msgs_dev(prm, cp, 0, C["msgs"].data_ptr(), ccap, C["offs"].data_ptr(),
                                      C["sizes"].data_ptr(), C["total"].data_ptr(), stream=st.cuda_stream)

        def host_call(k, p):
            s = sess[k]
            if k == "push_scan_cloud":
                a, b, _ = s.push_scan_cloud_msgs(pools[p], cnt, prm, cp, 0, rx_us=rxs[p], timing=timing,
                                                 msgs=h_msgs[0], cloud_msgs=h_msgs[1])
                return a["total_bytes"], b["total_bytes"]
            a, _ = s.push_laserscan_msgs(pools[p], cnt, prm, 0, rx_us=rxs[p], timing=timing, msgs=h_msgs[0],
                                         packed=True)
            if k == "floor":
                return a["total_bytes"], 0
            b = s.scan_cloud_msgs(prm, cp, 0, msgs=h_msgs[1], packed=True)
            return a["total_bytes"], b["total_bytes"]

        def timed_dev(k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                dev_call(k, step[k] % POOL)
                step[k] += 1
            e1.record(st)
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps

        totals = {}

        def timed_host(k):
            t0 = time.perf_counter()
            for _ in range(args.steps):
                totals[k] = host_call(k, step[k] % POOL)
                step[k] += 1
            return (time.perf_counter() - t0) / args.steps * 1e3

        rounds = {f"{form}_{k}": [] for form in ("dev", "host") for k in VARIANTS}
        for _ in range(args.warmup):
            for k in VARIANTS:
                timed_dev(k)
                timed_host(k)
        for _ in range(args.rounds):
            for k in VARIANTS:
                rounds[f"dev_{k}"].append(timed_dev(k))
            for k in VARIANTS:
                rounds[f"host_{k}"].append(timed_host(k))
        for s in sess.values():
            s.close()
        tables = NS * 12 + 8  # one set's offsets, sizes and total
        st_b, sc_b = totals["push_scan_cloud"]
        res["filtered" if filtered else "plain"] = {
            "ms_per_push": {k: float(np.median(v)) for k, v in rounds.items()},
            "d2h_bytes_last_push": {
                "floor": totals["floor"][0] + tables + 4 * n,
                "two_calls": sum(totals["two_calls"]) + 2 * tables + 4 * n,
                "push_scan_cloud": st_b + sc_b + 2 * tables + 4 * n},
            "scan_total_bytes": int(st_b), "cloud_total_bytes": int(sc_b), "rounds": rounds}
    ctx.close()
    return {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    res = {"gpu": gpu_info()}
    for sh in args.shapes.split(","):
        res[sh] = run_shape(R, torch, *SHAPES[sh], args)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
