"""The footprint stage of the per-stream LaserScan filters (rpl_capsule_stream_set_scan_footprints) on the shapes of
bench_stream_scan_filters.py (DESIGN.md 5.7.1); prints one JSON line.

Every variant is stamped rpl_capsule_stream_push_laserscan_msgs_dev on one CUDA stream, timed with CUDA events per push
(dense capsules, 0x85, Mode B; a pool of 8 pushes replayed in turn), each on its own session of the same streams:
  * no_flag: the call without RPL_FLAG_PER_STREAM_FILTERS;
  * neutral: the flag with every stream's entry enabled and removing nothing, and no footprint;
  * box: the neutral entries and one 4-vertex box per stream (a 0.6 x 0.4 m body about the lidar);
  * polygons_4x16: the neutral entries and four 16-vertex polygons per stream, placed so that most beams test all 64
    edges.
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


def footprints(R, n):
    box = R.scan_footprint([[(-0.3, -0.2), (0.3, -0.2), (0.3, 0.2), (-0.3, 0.2)]], pose=(0.1, 0.0, 0.0))
    rng = np.random.default_rng(1)
    polys = []
    for p in range(4):  # small stars off to the sides: few beams fall in one, so most test every polygon
        a = np.sort(rng.uniform(0, 2 * math.pi, 16))
        cx, cy = 3.0 * math.cos(p * math.pi / 2 + 0.4), 3.0 * math.sin(p * math.pi / 2 + 0.4)
        polys.append([(cx + q * math.cos(t), cy + q * math.sin(t)) for t, q in zip(a, rng.uniform(0.2, 0.6, 16))])
    many = R.scan_footprint(polys, invert=[0, 0, 0, 0], pose=(0.0, 0.0, 0.0))
    return {"box": [box] * n, "polygons_4x16": [many] * n}


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
    cap = NS * ((288 + 32 + 8 * max_nodes + 4 + 15) // 16 * 16)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    plain = R.scan_params(0, 0, 0, 1)
    flag = R.scan_params(0, 0, 0, 1, R.FLAG_PER_STREAM_FILTERS)

    def variant(flagged, fps=None):
        s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
        if flagged:
            s.set_scan_filters([R.scan_filter_settings()] * n)
        if fps is not None:
            s.set_scan_footprints(fps)
        prm = flag if flagged else plain
        step = [0]

        def run():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                p = step[0] % POOL
                step[0] += 1
                s.push_laserscan_msgs_dev(pools[p].data_ptr(), cnt.data_ptr(), prm, 0, d_msgs.data_ptr(), cap,
                                          d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(), d_sps.data_ptr(),
                                          rx_us=rxs[p].data_ptr(), timing=timing, stream=st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps
        return s, run

    built = {"no_flag": variant(False), "neutral": variant(True)}
    for k, t in footprints(R, n).items():
        built[k] = variant(True, t)
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
