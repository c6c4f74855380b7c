"""What per-stream lidar settings (rpl_capsule_stream_set_lidars + RPL_FLAG_PER_STREAM) cost a device push; prints one
JSON line.

Shape: the chain shape of bench.py, 512 dense-capsule streams (0x85) x 4096 capsules per push (about 51 revolutions of
3200 nodes per stream), max_nodes 4096, max_scans 56.  push_dev is timed with CUDA events, in rounds that alternate
the four variants:
  noflag     one session of 512 streams, uniform params, no flag;
  uniform    the same session with the flag and every table entry equal to those params;
  mixed      the flag with odd streams in Mode A and inverted, even streams in Mode B (one launch of each mode);
  two        the work of `mixed` as two uniform sessions of 256 streams (even streams Mode B, odd Mode A inverted).
Every push replays the same capsules, so each stream continues with one angular jump per push.  The medians over the
rounds are reported, with the GPU's name and power limit read in the same run.
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

N_STREAMS, CAPS, MAX_NODES, MAX_SCANS = 512, 4096, 4096, 56


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=20, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the H100 path only")
    name, power = gpu_info()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    caps = feed(N_STREAMS, CAPS)
    d_caps = torch.from_numpy(caps).to(dev)
    d_even = d_caps[0::2].contiguous()
    d_odd = d_caps[1::2].contiguous()
    d_cnt = torch.full((N_STREAMS,), CAPS, dtype=torch.int32, device=dev)
    NS = N_STREAMS * MAX_SCANS
    r = torch.empty((NS, MAX_NODES), device=dev)
    it = torch.empty((NS, MAX_NODES), device=dev)
    bc = torch.empty(NS, dtype=torch.int32, device=dev)
    inc = torch.empty(NS, device=dev)
    sps = torch.empty(N_STREAMS, dtype=torch.int32, device=dev)
    half = NS // 2
    ctx = R.Context(0, MAX_NODES, NS)

    base = R.scan_params(1, 0, 0, 1)
    per = R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM)
    t31 = R.Timing(31, 0, 0, 0)
    sessions = {k: R.DenseStreamSession(ctx, N_STREAMS, CAPS, MAX_NODES, MAX_SCANS) for k in ("noflag", "uniform", "mixed")}
    sessions["uniform"].set_lidars([R.lidar_settings(1, 0, 0, t31)] * N_STREAMS)
    sessions["mixed"].set_lidars([R.lidar_settings(1, s & 1, s & 1, t31) for s in range(N_STREAMS)])
    two = [R.DenseStreamSession(ctx, N_STREAMS // 2, CAPS, MAX_NODES, MAX_SCANS) for _ in range(2)]
    two_params = [R.scan_params(1, 0, 0, 1), R.scan_params(1, 1, 1, 1)]

    def push(sess, d_in, params, o=0, nsl=NS):
        sess.push_dev(d_in.data_ptr(), d_cnt.data_ptr(), params, r[o:o + nsl].data_ptr(), it[o:o + nsl].data_ptr(),
                      bc[o:].data_ptr(), inc[o:].data_ptr(), sps.data_ptr(), stream=st.cuda_stream)

    steps = {
        "noflag": lambda: push(sessions["noflag"], d_caps, base),
        "uniform": lambda: push(sessions["uniform"], d_caps, per),
        "mixed": lambda: push(sessions["mixed"], d_caps, per),
        "two": lambda: (push(two[0], d_even, two_params[0], 0, half), push(two[1], d_odd, two_params[1], half, half)),
    }

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(n):
            fn()
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / n

    torch.cuda.synchronize()
    for fn in steps.values():
        timed(fn, args.warmup)
    rounds = {k: [] for k in steps}
    for _ in range(args.rounds):
        for k, fn in steps.items():
            rounds[k].append(timed(fn, args.steps))
    scans = int(sps.sum().item())  # of the last push (the second uniform session's half)
    med = {k: float(np.median(v)) for k, v in rounds.items()}
    print(json.dumps({
        "gpu": name, "power_limit": power, "n_streams": N_STREAMS, "capsules_per_push": CAPS, "max_nodes": MAX_NODES,
        "max_scans": MAX_SCANS, "scans_last_push_of_one_half": scans,
        "push_dev_ms": {f"{k}_median": v for k, v in med.items()},
        "mixed_over_noflag": med["mixed"] / med["noflag"], "uniform_over_noflag": med["uniform"] / med["noflag"],
        "two_over_mixed": med["two"] / med["mixed"], "rounds_ms": rounds,
    }))
    for s in (*sessions.values(), *two):
        s.close()
    ctx.close()


if __name__ == "__main__":
    main()
