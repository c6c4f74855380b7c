"""Clouds projected from the LaserScans (rpl_capsule_stream_scan_cloud_msgs_dev) next to the LaserScan messages alone
(rpl_capsule_stream_laserscan_msgs_dev), on the dense shapes of bench_stream_scan_filters.py (DESIGN.md 5.7.1);
prints one JSON line.

Each shape's session takes one stamped push of the capsules of POOL of the shape's pushes (dense, 0x85, Mode B), so
that the push publishes scans on every stream; every variant is then the message call over that push's scans, on one
CUDA stream, timed with CUDA events over --steps calls:
  * laserscan_msgs: laserscan_msgs_dev;
  * scan_cloud_default: scan_cloud_msgs_dev with laser_geometry's default channels (intensity, index);
  * scan_cloud_all: scan_cloud_msgs_dev with all four channels;
  * laserscan_msgs_filtered, scan_cloud_filtered: the same two with RPL_FLAG_PER_STREAM_FILTERS, every stream running
    the whole filter chain and a footprint box.
Both calls recompute the LaserScans of the push; the difference is the projection's cost.  The variants alternate in
rounds within one run; each figure is the median over the rounds, with the rounds listed.  The GPU's name, power
limit and SM clocks are read in the same run.
"""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed  # noqa: E402
from bench_stream_scan_filters import POOL, SHAPES, gpu_info  # noqa: E402


def run_shape(R, torch, n, units, max_nodes, ms, args):
    units *= POOL
    data = feed(n, units)
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    caps = torch.from_numpy(np.ascontiguousarray(data)).to(dev)
    rx = torch.from_numpy((10_000_000 + np.arange(units, dtype=np.uint64) * 250)[None, :].repeat(n, 0)
                          .view(np.int64)).to(dev)
    cnt = torch.full((n,), units, dtype=torch.int32, device=dev)
    ctx = R.Context(0, max_nodes, n * ms)
    NS = n * ms
    cap = NS * ((288 + 192 + 28 * max_nodes + 1 + 15) // 16 * 16)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    plain = R.scan_params(0, 0, 0, 1)
    flag = R.scan_params(0, 0, 0, 1, R.FLAG_PER_STREAM_FILTERS)
    s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
    s.set_frames([f"laser_{k}" for k in range(n)])
    s.set_scan_filters([R.scan_filter_settings(mask=[(2.8, 3.4)], range_lo=0.15, range_hi=12.0, intensity_min=1.0,
                                               speckle_window=3, speckle_min_neighbours=2, speckle_max_diff=0.05,
                                               shadow_window=8, shadow_angle=math.radians(10))] * n)
    s.set_scan_footprints([R.scan_footprint([[(-0.4, -0.3), (0.4, -0.3), (0.4, 0.3), (-0.4, 0.3)]])] * n)
    s.push_laserscan_msgs_dev(caps.data_ptr(), cnt.data_ptr(), plain, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(),
                              d_sz.data_ptr(), d_tot.data_ptr(), d_sps.data_ptr(), rx_us=rx.data_ptr(),
                              timing=R.Timing(31, 0, 0, 0), stream=st.cuda_stream)
    st.synchronize()
    default, every = R.scan_cloud_params(), R.scan_cloud_params(0x0F)
    calls = {
        "laserscan_msgs": lambda: s.laserscan_msgs_dev(plain, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(),
                                                       d_sz.data_ptr(), d_tot.data_ptr(), stream=st.cuda_stream),
        "scan_cloud_default": lambda: s.scan_cloud_msgs_dev(plain, default, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(),
                                                            d_sz.data_ptr(), d_tot.data_ptr(), stream=st.cuda_stream),
        "scan_cloud_all": lambda: s.scan_cloud_msgs_dev(plain, every, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(),
                                                        d_sz.data_ptr(), d_tot.data_ptr(), stream=st.cuda_stream),
        "laserscan_msgs_filtered": lambda: s.laserscan_msgs_dev(flag, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(),
                                                                d_sz.data_ptr(), d_tot.data_ptr(),
                                                                stream=st.cuda_stream),
        "scan_cloud_filtered": lambda: s.scan_cloud_msgs_dev(flag, default, 0, d_msgs.data_ptr(), cap,
                                                             d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(),
                                                             stream=st.cuda_stream),
    }

    def timed(call):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            call()
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for _ in range(args.warmup):
        for c in calls.values():
            timed(c)
    rounds = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, c in calls.items():
            rounds[k].append(timed(c))
    scans = int((d_sz.cpu().numpy() > 0).sum())
    points = int(d_tot.cpu().numpy()[0])
    s.close()
    ctx.close()
    return {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms,
            "messages": scans, "last_total_bytes": points,
            "ms_per_call": {k: float(np.median(v)) for k, v in rounds.items()}, "rounds": rounds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed calls per variant and round")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
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
