"""Moving a whole fleet between stream sessions (rpl_capsule_stream_export / _import); prints one JSON line.

Workload: 512 streams in a 0x81 byte session, each holding an open revolution capped at max_nodes (a first push of
max_nodes + 100 records behind one scan start), at max_nodes 4096 and 8192 -- the largest records a session holds.
Per shape: the wall time of one export of all 512 streams and of one import of those records into a second session of
the same shape (host clock around each synchronous call, median of --reps), the pack and unpack kernels' own times
(the CUDA profiler's kernel records, in a pass of their own, median), the record bytes, and next to them the wall time
of what moving replaces: destroying the session and creating a fresh one (which loses every stream's state).  The GPU's
name and power limit are part of the output.
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

from bench_stream_msgs import gpu_info  # noqa: E402

N_STREAMS = 512
MAX_SCANS = 4


def open_revolution_bytes(n_rec, seed=1):
    """0x81 records: one scan start, then n_rec - 1 records of one revolution that never closes"""
    rng = np.random.default_rng(seed)
    rec = np.empty((n_rec, 5), np.uint8)
    start = np.zeros(n_rec, np.uint8)
    start[0] = 1
    rec[:, 0] = (rng.integers(0, 64, n_rec).astype(np.uint8) << 2) | ((1 - start) << 1) | start
    w = ((np.arange(n_rec) * (360 * 64) // (n_rec + 1)) << 1) | 1
    rec[:, 1], rec[:, 2] = w & 0xFF, w >> 8
    dist = rng.integers(4, 65536, n_rec)
    rec[:, 3], rec[:, 4] = dist & 0xFF, dist >> 8
    return rec.reshape(-1)


def run_shape(R, torch, max_nodes, reps):
    n_rec = max_nodes + 100
    stride = n_rec * 5
    data = np.tile(open_revolution_bytes(n_rec), (N_STREAMS, 1))
    ctx = R.Context(0, max_nodes, N_STREAMS * MAX_SCANS)
    prm = R.scan_params(1, 0, 0, 1)
    a = R.NormalStreamSession(ctx, N_STREAMS, stride, max_nodes, MAX_SCANS)
    b = R.NormalStreamSession(ctx, N_STREAMS, stride, max_nodes, MAX_SCANS)
    a.push(data, np.full(N_STREAMS, stride, np.uint32), prm)
    open_nodes = a.state()[0]
    streams = np.arange(N_STREAMS, dtype=np.uint32)
    recs, offs = a.export_streams(streams)  # warm-up: module load and the staging allocations
    b.import_streams(streams, recs, offs)
    exp, imp, rec = [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        recs, offs = a.export_streams(streams)
        t1 = time.perf_counter()
        b.import_streams(streams, recs, offs)
        t2 = time.perf_counter()
        exp.append(t1 - t0)
        imp.append(t2 - t1)
    for _ in range(reps):
        t0 = time.perf_counter()
        b.close()
        b = R.NormalStreamSession(ctx, N_STREAMS, stride, max_nodes, MAX_SCANS)
        rec.append(time.perf_counter() - t0)
    # the kernels' own times, from the profiler's kernel records in a pass of their own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            recs, offs = a.export_streams(streams)
            b.import_streams(streams, recs, offs)
    kern = {"pack": [], "unpack": []}
    for e in prof.events():
        if "stream_pack_kernel" in e.name:
            kern["pack"].append(e.time_range.elapsed_us())
        elif "stream_unpack_kernel" in e.name:
            kern["unpack"].append(e.time_range.elapsed_us())
    total = int(recs.size)
    med = lambda x: float(np.median(x))  # noqa: E731
    pack_us, unpack_us = med(kern["pack"]) if kern["pack"] else None, med(kern["unpack"]) if kern["unpack"] else None
    out = {
        "max_nodes": max_nodes, "open_nodes_min": int(open_nodes.min()), "open_nodes_max": int(open_nodes.max()),
        "record_bytes_total": total, "record_bytes_per_stream": total // N_STREAMS,
        "export_wall_ms": round(1e3 * med(exp), 3), "import_wall_ms": round(1e3 * med(imp), 3),
        "move_wall_ms": round(1e3 * (med(exp) + med(imp)), 3),
        "pack_kernel_us": None if pack_us is None else round(pack_us, 1),
        "unpack_kernel_us": None if unpack_us is None else round(unpack_us, 1),
        # bytes each kernel reads and writes: the records once each way
        "pack_GBps": None if not pack_us else round(2 * total / pack_us / 1e3, 1),
        "unpack_GBps": None if not unpack_us else round(2 * total / unpack_us / 1e3, 1),
        "recreate_wall_ms": round(1e3 * med(rec), 3),
    }
    a.close()
    b.close()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "n_streams": N_STREAMS, "reps": args.reps,
           "shapes": [run_shape(R, torch, m, args.reps) for m in (4096, 8192)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
