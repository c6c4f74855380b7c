"""Footprints in the clouds (RPL_CLOUD_PER_STREAM_FOOTPRINTS) on the shapes of bench_stream_scan_filters.py
(DESIGN.md 5.7.1 "Footprints in the clouds"); prints one JSON line.

Every variant is stamped rpl_capsule_stream_push_cloud_msgs_dev with RPL_CLOUD_PER_STREAM_CHAIN on one CUDA stream,
every stream's chain SOR 8 + 5 cm voxels (the route the fused shared-memory kernel takes), timed with CUDA events per
push (dense capsules, 0x85, Mode B; a pool of 8 pushes replayed in turn), each on its own session of the same streams:
  * no_flag: the call without RPL_CLOUD_PER_STREAM_FOOTPRINTS;
  * empty: the flag, every stream's footprint without polygons (expected equal to no_flag);
  * box: the flag and one 4-vertex box per stream (a 0.6 x 0.4 m body about the lidar);
  * no_fused: no_flag with RPL_CLOUD_NO_FUSED: the cost of leaving the fused kernel, without the footprint pass;
  * polygons_4x16: the flag and four 16-vertex polygons per stream, placed so that most points test all 64 edges.
The variants alternate in rounds within one run; each figure is the median over the rounds, with the rounds listed.
The GPU's name, power limit and SM clocks are read in the same run.
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
from bench_stream_scan_footprints import footprints  # noqa: E402


def run_shape(R, torch, n, units, max_nodes, ms, args):
    data = feed(n, units * POOL)  # [n, units * POOL, 84]
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    pools = [torch.from_numpy(np.ascontiguousarray(data[:, p * units:(p + 1) * units])).to(dev) for p in range(POOL)]
    rxs = [torch.from_numpy((10_000_000 + 100_000 * p + np.arange(units, dtype=np.uint64) * 250)[None, :]
                            .repeat(n, 0).view(np.int64)).to(dev) for p in range(POOL)]
    cnt = torch.full((n,), units, dtype=torch.int32, device=dev)
    timing = R.Timing(31, 0, 0, 0)
    ctx = R.Context(0, max_nodes, n * ms)
    NS = n * ms
    cap = NS * ((288 + 116 + 16 * max_nodes + 1 + 15) // 16 * 16)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    chain = [R.cloud_settings(0.15, 40.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)] * n

    def variant(flags, fps=None):
        s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
        s.set_frames(["laser"] * n, np.full(n, 40.0, np.float32))
        s.set_clouds(chain)
        if fps is not None:
            s.set_scan_footprints(fps)
        prm = R.cloud_params(0.15, 40.0, 0.0, flags=R.CLOUD_PER_STREAM_CHAIN | flags)
        step = [0]

        def run():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                p = step[0] % POOL
                step[0] += 1
                s.push_cloud_msgs_dev(pools[p].data_ptr(), cnt.data_ptr(), prm, 0, d_msgs.data_ptr(), cap,
                                      d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(), d_sps.data_ptr(),
                                      rx_us=rxs[p].data_ptr(), timing=timing, stream=st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps
        return s, run

    F = R.CLOUD_PER_STREAM_FOOTPRINTS
    fps = footprints(R, n)
    built = {"no_flag": variant(0), "empty": variant(F, [R.scan_footprint()] * n), "box": variant(F, fps["box"]),
             "no_fused": variant(R.CLOUD_NO_FUSED), "polygons_4x16": variant(F, fps["polygons_4x16"])}
    runs = {k: r for k, (_, r) in built.items()}
    for _ in range(args.warmup):
        for r in runs.values():
            r()
    rounds = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, r in runs.items():
            rounds[k].append(r())
    for s, _ in built.values():
        s.close()
    ctx.close()
    return {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms,
            "ms_per_push": {k: float(np.median(v)) for k, v in rounds.items()}, "rounds": rounds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    res = {"gpu": gpu_info()}
    for s in args.shapes.split(","):
        res[s] = run_shape(R, torch, *SHAPES[s], args)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
