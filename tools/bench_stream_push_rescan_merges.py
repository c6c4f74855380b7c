"""Merged scans from the push, rpl_capsule_stream_push_rescan_merge_msgs_dev, against push_rescan_msgs_dev on the
dense shapes of bench_stream_rescans.py (DESIGN.md 5.7.1 "Merged scans from the push"); prints one JSON line.

Every shape has one session per variant, each with its streams mounted by a 3-D transform into base_link and
re-gridded onto pointcloud_to_laserscan's default 360-beam grid:
  push_rescan       push_rescan_msgs_dev, no window;
  merge_g2_age0     the merge push, streams 2j and 2j + 1 in group j, max_age 0, no window;
  merge_g4_age0     the same with groups of four;
  merge_g2_median5  merge_g2_age0 with a median over 5 revolutions on every stream;
  merge_g4_median5  merge_g4_age0 with the same windows.
Each variant's pushes take the next of POOL stamped dense pushes (0x85, Mode B) in turn.  In every round the variants
are timed one after the other, `steps` frames each, with CUDA events on one CUDA stream; each figure is the median of
the rounds' ms per frame, with the rounds listed.  The GPU's name, power limit and SM clocks are read in the same run.
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

VARIANTS = {"push_rescan": (0, 1), "merge_g2_age0": (2, 1), "merge_g4_age0": (4, 1), "merge_g2_median5": (2, 5),
            "merge_g4_median5": (4, 5)}  # (group size, 0: no merge; median window)


def run_shape(R, torch, n, units, max_nodes, ms, args):
    NS = n * ms
    data = feed(n, units * POOL)
    pools = [np.ascontiguousarray(data[:, p * units:(p + 1) * units]) for p in range(POOL)]
    rxs = [(10_000_000 + 100_000 * p + np.arange(units, dtype=np.uint64) * 250)[None, :].repeat(n, 0)
           for p in range(POOL)]
    cnt = np.full(n, units, np.uint32)
    timing = R.Timing(31, 0, 0, 0)
    ctx = R.Context(0, max_nodes, NS)
    cp = R.scan_cloud_params(R.SCAN_CLOUD_PER_STREAM_TRANSFORMS)
    rng = np.random.default_rng(5)

    def mount(k):  # a lidar on a mast, yawed, pitched and rolled a little
        roll, pitch, yaw = rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(-math.pi, math.pi)
        cr, sr, cp_, sp, cy, sy = (math.cos(roll / 2), math.sin(roll / 2), math.cos(pitch / 2), math.sin(pitch / 2),
                                   math.cos(yaw / 2), math.sin(yaw / 2))
        q = (sr * cp_ * cy - cr * sp * sy, cr * sp * cy + sr * cp_ * sy, cr * cp_ * sy - sr * sp * cy,
             cr * cp_ * cy + sr * sp * sy)
        return R.scan_cloud_transform((0.3 + 0.01 * k, -0.2, 0.45), q)

    mounts = [mount(j) for j in range(n)]
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    d_pool = [torch.from_numpy(x).to(dev) for x in pools]
    d_rx = [torch.from_numpy(x.view(np.int64)).to(dev) for x in rxs]
    d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    prm = R.scan_params(0, 0, 0, 1)

    def out(c):
        t = dict(msgs=torch.empty(c, dtype=torch.uint8, device=dev), offs=torch.empty(NS, dtype=torch.int64, device=dev),
                 sizes=torch.empty(NS, dtype=torch.int32, device=dev), total=torch.empty(1, dtype=torch.int64, device=dev))
        t["out"] = R.MsgsOut(t["msgs"].data_ptr(), c, t["offs"].data_ptr(), t["sizes"].data_ptr(), t["total"].data_ptr())
        return t

    scans = out(NS * ((288 + 32 + 8 * max_nodes + 4 + 15) // 16 * 16))
    rescans = out(NS * ((288 + 36 + 4 * 360 + 15) // 16 * 16))
    merged = out(n * ((288 + 36 + 4 * 360 + 15) // 16 * 16))
    sessions, groups = {}, {}
    for k, (size, obs) in VARIANTS.items():
        s = R.DenseStreamSession(ctx, n, units, max_nodes, ms)
        s.set_frames([f"laser_{j}" for j in range(n)])
        s.set_scan_cloud_transforms(mounts, ["base_link"] * n)
        s.set_rescans([R.rescan_settings(range_min=0.15, range_max=40.0, min_height=-0.5, max_height=1.5)] * n)
        if obs > 1:
            s.set_rescan_windows([R.rescan_window(obs, "median")] * n)
        if size:
            groups[k] = -(-n // size)
            s.set_rescan_merges([j // size for j in range(n)], [0] * groups[k])
        sessions[k] = s
    step = {k: 0 for k in VARIANTS}

    def frame(k):
        s, p = sessions[k], step[k] % POOL
        step[k] += 1
        if k in groups:
            s.push_rescan_merge_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, cp, 0, scans["out"],
                                         rescans["out"], merged["out"], d_sps.data_ptr(), rx_us=d_rx[p].data_ptr(),
                                         timing=timing, stream=st.cuda_stream)
        else:
            s.push_rescan_msgs_dev(d_pool[p].data_ptr(), d_cnt.data_ptr(), prm, cp, 0, scans["out"], rescans["out"],
                                   d_sps.data_ptr(), rx_us=d_rx[p].data_ptr(), timing=timing, stream=st.cuda_stream)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            frame(k)
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    rounds = {k: [] for k in VARIANTS}
    totals = {}
    for r in range(args.warmup + args.rounds):
        for k in VARIANTS:
            t = timed(k)
            if r >= args.warmup:
                rounds[k].append(t)
                totals[k] = [int(rescans["total"].cpu().numpy()[0]),
                             int(merged["total"].cpu().numpy()[0]) if k in groups else 0]
    for s in sessions.values():
        s.close()
    ctx.close()
    return {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms,
            "ms_per_frame": {k: float(np.median(v)) for k, v in rounds.items()},
            "rescan_and_merged_total_bytes": totals,
            "rounds": rounds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed frames per variant and round")
    ap.add_argument("--rounds", type=int, default=7)
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
