"""Per-stream LaserScan filters (rpl_capsule_stream_set_scan_filters, RPL_FLAG_PER_STREAM_FILTERS) on the dense shapes
of bench_stream_clouds.py (DESIGN.md 5.7.1); prints one JSON line.

Every variant is stamped rpl_capsule_stream_push_laserscan_msgs_dev on one CUDA stream, timed with CUDA events per push
(dense capsules, 0x85, Mode B; a pool of 8 pushes replayed in turn), each on its own session of the same streams:
  * no_flag: the call without the flag;
  * all_disabled: the flag with every stream's entry disabled (no filter launch);
  * full_chain: the flag with every stream running the whole chain (a masked sector, range window, intensity floor,
    speckle window 3, veiling window 8);
  * mixed: the flag on a fleet cycling through the whole chain, speckle only, veiling only and disabled.
The variants alternate in rounds within one run; each figure is the median over the rounds, with the rounds listed.
The GPU's name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed  # noqa: E402

SHAPES = {"aggregator": (256, 320, 4096, 4), "live": (512, 80, 8192, 2)}
POOL = 8


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (x.strip() for x in line.split(","))))
    except Exception:  # noqa: BLE001
        return {"name": "unknown"}


def tables(R, n):
    chain = R.scan_filter_settings(mask=[(2.8, 3.4)], range_lo=0.15, range_hi=12.0, intensity_min=1.0,
                                   speckle_window=3, speckle_min_neighbours=2, speckle_max_diff=0.05, shadow_window=8,
                                   shadow_angle=math.radians(10))
    speckle = R.scan_filter_settings(speckle_window=2, speckle_min_neighbours=1, speckle_max_diff=0.05)
    veiling = R.scan_filter_settings(shadow_window=8, shadow_angle=math.radians(10))
    off = R.scan_filter_settings(enabled=False)
    cycle = [chain, speckle, veiling, off]
    return {"all_disabled": [off] * n, "full_chain": [chain] * n, "mixed": [cycle[s % 4] for s in range(n)]}


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

    def variant(table):
        s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
        if table is not None:
            s.set_scan_filters(table)
        prm = plain if table is None else flag
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

    built = {"no_flag": variant(None)}
    for k, t in tables(R, n).items():
        built[k] = variant(t)
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
