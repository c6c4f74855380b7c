"""Per-stream clouds (rpl_capsule_stream_set_clouds, RPL_CLOUD_PER_STREAM_CHAIN) on the dense shapes of
bench_stream_push_cloud_msgs.py; prints one JSON line.

Every variant is stamped rpl_capsule_stream_push_cloud_msgs_dev on one CUDA stream, timed with CUDA events per push
(dense capsules, 0x85; a pool of 8 pushes replayed in turn):
  * uniform: the flagless call with SOR 8 + 5 cm voxels against the flagged call with every stream's entry equal to it;
  * fleet: one session whose streams cycle through window only, 5 cm voxels, SOR 8 + 5 cm voxels and no cloud (a
    quarter of the streams), against one session per configuration holding that configuration's streams (the streams
    without a cloud are in none of them: that split decodes less than the fleet does);
  * half off: the fleet's three configurations on every stream, against the same with every second stream disabled.
The variants of a comparison alternate in rounds within one run; each figure is the median over the rounds, with the
rounds listed.  The GPU's name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
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


def configs(R):
    return [R.cloud_settings(0.15, 40.0, 0.0),
            R.cloud_settings(0.15, 40.0, 0.0, voxel_size=0.05),
            R.cloud_settings(0.15, 40.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0)]


def params_of(R, e, flags=0):
    return R.cloud_params(e.range_min, e.range_max, e.intensity_min, e.voxel_size, e.sor_k, e.sor_alpha, 0, flags)


def run_shape(R, torch, n, units, max_nodes, ms, args):
    data = feed(n, units * POOL)  # [n, units * POOL, 84]
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    pools = [torch.from_numpy(np.ascontiguousarray(data[:, p * units:(p + 1) * units])).to(dev) for p in range(POOL)]
    rxs = [torch.from_numpy((10_000_000 + 100_000 * p + np.arange(units, dtype=np.uint64) * 250)[None, :]
                            .repeat(n, 0).view(np.int64)).to(dev) for p in range(POOL)]
    timing = R.Timing(31, 0, 0, 0)
    ctx = R.Context(0, max_nodes, n * ms)
    NS = n * ms
    cap = NS * ((288 + 116 + 16 * max_nodes + 1 + 15) // 16 * 16)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    d_sps = torch.empty(n, dtype=torch.int32, device=dev)
    cfg = configs(R)
    off = R.cloud_settings(enabled=False)
    chain = R.CLOUD_PER_STREAM_CHAIN

    def session(streams, table=None):
        """a session of these streams (their slice of the feed) pushed with table / params"""
        s = R.DenseStreamSession(ctx, len(streams), units, max_nodes, ms)
        if table is not None:
            s.set_clouds(table)
        idx = torch.tensor(streams, device=dev)
        cnt = torch.full((len(streams),), units, dtype=torch.int32, device=dev)
        pool = [p.index_select(0, idx).contiguous() for p in pools] if len(streams) < n else pools
        rx = [x.index_select(0, idx).contiguous() for x in rxs] if len(streams) < n else rxs
        return s, cnt, pool, rx

    def variant(parts):
        """parts: [(session, cnt, pool, rx, params)] pushed one after the other per step"""
        step = [0]

        def run():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.steps):
                p = step[0] % POOL
                step[0] += 1
                for s, cnt, pool, rx, prm in parts:
                    s.push_cloud_msgs_dev(pool[p].data_ptr(), cnt.data_ptr(), prm, 0, d_msgs.data_ptr(), cap,
                                          d_off.data_ptr(), d_sz.data_ptr(), d_tot.data_ptr(), d_sps.data_ptr(),
                                          rx_us=rx[p].data_ptr(), timing=timing, stream=st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps
        return run

    everyone = list(range(n))
    built = []

    def part(streams, prm, table=None):
        s = session(streams, table)
        built.append(s[0])
        return (*s, prm)

    fleet_table = [off if s % 4 == 3 else cfg[s % 4] for s in range(n)]
    half_table = [off if s % 2 else cfg[(s // 2) % 3] for s in range(n)]
    full_table = [cfg[(s // 2) % 3] for s in range(n)]
    comparisons = {
        "uniform": {"flagless": [part(everyone, params_of(R, cfg[2]))],
                    "uniform_table": [part(everyone, R.cloud_params(flags=chain), [cfg[2]] * n)]},
        "fleet": {"one_session": [part(everyone, R.cloud_params(flags=chain), fleet_table)],
                  "session_per_config": [part([s for s in everyone if s % 4 == c], params_of(R, cfg[c]))
                                         for c in range(3)]},
        "half_off": {"all_enabled": [part(everyone, R.cloud_params(flags=chain), full_table)],
                     "half_disabled": [part(everyone, R.cloud_params(flags=chain), half_table)]},
    }
    res = {"n_streams": n, "units_per_push": units, "max_nodes": max_nodes, "max_scans": ms}
    for name, variants in comparisons.items():
        runs = {k: variant(v) for k, v in variants.items()}
        for _ in range(args.warmup):
            for r in runs.values():
                r()
        rounds = {k: [] for k in runs}
        for _ in range(args.rounds):
            for k, r in runs.items():
                rounds[k].append(r())
        res[name] = {"ms_per_push": {k: float(np.median(v)) for k, v in rounds.items()}, "rounds": rounds}
    for s in built:
        s.close()
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

    res = {"gpu": gpu_info()}
    for s in args.shapes.split(","):
        res[s] = run_shape(R, torch, *SHAPES[s], args)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
