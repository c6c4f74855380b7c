"""Packed LaserScan messages of a stream session (rpl_capsule_stream_laserscan_msgs[_dev]) against the padded arrays of
the push; prints one JSON line.

Shape: a multi-lidar aggregator of 256 dense-capsule streams (0x85), each push one receive period of 320 capsules per
stream (4 revolutions of about 3200 nodes), max_nodes 4096, max_scans 4.  Reported per push:
  * bytes copied device-to-host: the packed messages (total_bytes plus the two tables) against the padded outputs of a
    host push ([n_streams * max_scans][max_nodes] ranges and intensities);
  * call time of a stamped host push + laserscan_msgs against the stamped host push alone (host buffers, synchronous:
    wall time), and of push_ts_dev + laserscan_msgs_dev against push_ts_dev alone (device buffers: CUDA events).
Pushes continue the streams, so every push publishes 4 revolutions per stream; the variants alternate in rounds within
one run.  The GPU's name and power limit are part of the output.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed  # noqa: E402

N_STREAMS, CAPS, MAX_NODES, MAX_SCANS = 256, 320, 4096, 4


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=20).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in q.split(","))
        return name, power
    except Exception:  # noqa: BLE001
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    n_push = 8  # a pool of pushes, replayed in turn (the wrap is one jump in angle per 8 pushes)
    caps = feed(N_STREAMS, CAPS * n_push)
    cnt = np.full(N_STREAMS, CAPS, np.uint32)
    prm = R.scan_params(1, 0, 0, 1)
    timing = R.Timing(31, 0, 0, 0)
    ctx = R.Context(0, MAX_NODES, N_STREAMS * MAX_SCANS)
    sess = R.DenseStreamSession(ctx, N_STREAMS, CAPS, MAX_NODES, MAX_SCANS)
    NS = N_STREAMS * MAX_SCANS
    out = {k: R.host_alloc(n).view(dt).reshape(shape) for k, n, dt, shape in (
        ("ranges", NS * MAX_NODES * 4, np.float32, (NS, MAX_NODES)),
        ("intensities", NS * MAX_NODES * 4, np.float32, (NS, MAX_NODES)),
        ("beam_counts", NS * 4, np.uint32, (NS,)), ("angle_increment", NS * 4, np.float32, (NS,)),
        ("scans_per_stream", N_STREAMS * 4, np.uint32, (N_STREAMS,)), ("scan_begin_ts_us", NS * 8, np.uint64, (NS,)))}
    msgs = R.host_alloc(NS * (288 + 36 + 8 * MAX_NODES + 16)).view(np.uint8)
    t = [0]

    def push_host():
        p = t[0] % n_push
        t[0] += 1
        rx = (10_000_000 + 80_000 * p + np.arange(CAPS, dtype=np.uint64) * 250)[None, :].repeat(N_STREAMS, 0)
        sess.push(np.ascontiguousarray(caps[:, p * CAPS:(p + 1) * CAPS]), cnt, prm, out=out, rx_us=rx, timing=timing)

    got = {}

    def run_host(with_msgs):
        dt = 0.0
        for _ in range(args.steps):
            t0 = time.perf_counter()
            push_host()
            if with_msgs:
                got["last"] = sess.laserscan_msgs(prm, 0, msgs=msgs, packed=True)
            dt += time.perf_counter() - t0
        return dt / args.steps * 1e3

    for _ in range(args.warmup):
        push_host()
        sess.laserscan_msgs(prm, 0, msgs=msgs, packed=True)
    host = {"push": [], "push_msgs": []}
    for _ in range(args.rounds):
        host["push"].append(run_host(False))
        host["push_msgs"].append(run_host(True))

    # device forms
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    d_caps = torch.from_numpy(caps).to(dev)  # [n_streams, CAPS * n_push, 84]
    d_cnt = torch.from_numpy(cnt.view(np.int32)).to(dev)
    d_rx = torch.arange(CAPS * N_STREAMS, dtype=torch.int64, device=dev).reshape(N_STREAMS, CAPS) * 250 + 10_000_000
    r = torch.empty((NS, MAX_NODES), device=dev)
    it = torch.empty((NS, MAX_NODES), device=dev)
    bc = torch.empty(NS, dtype=torch.int32, device=dev)
    inc = torch.empty(NS, device=dev)
    sps = torch.empty(N_STREAMS, dtype=torch.int32, device=dev)
    ts = torch.empty(NS, dtype=torch.int64, device=dev)
    cap = NS * (288 + 36 + 8 * MAX_NODES + 16)
    d_msgs = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_sz = torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.empty(1, dtype=torch.int64, device=dev)
    sess2 = R.DenseStreamSession(ctx, N_STREAMS, CAPS, MAX_NODES, MAX_SCANS)
    k = [0]

    d_push = torch.empty((N_STREAMS, CAPS, 84), dtype=torch.uint8, device=dev)

    def push_dev():
        p = k[0] % n_push
        k[0] += 1
        with torch.cuda.stream(st):
            d_push.copy_(d_caps[:, p * CAPS:(p + 1) * CAPS].reshape(N_STREAMS, CAPS, 84))
        sess2.push_dev(d_push.data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                       inc.data_ptr(), sps.data_ptr(), stream=st.cuda_stream, rx_us=d_rx.data_ptr(), timing=timing,
                       scan_begin_ts_us=ts.data_ptr())

    def run_dev(with_msgs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            push_dev()
            if with_msgs:
                sess2.laserscan_msgs_dev(prm, 0, d_msgs.data_ptr(), cap, d_off.data_ptr(), d_sz.data_ptr(),
                                         d_tot.data_ptr(), stream=st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for _ in range(args.warmup):
        run_dev(True)
    devt = {"push_dev": [], "push_dev_msgs": []}
    for _ in range(args.rounds):
        devt["push_dev"].append(run_dev(False))
        devt["push_dev_msgs"].append(run_dev(True))
    # both variants include the device copy that lays each push's capsules out as [n_streams][CAPS][84]

    last = got["last"]
    n_msgs = int((last["msg_sizes"] > 0).sum())
    padded = 2 * NS * MAX_NODES * 4 + NS * 4 * 2 + NS * 8 + N_STREAMS * 4
    packed = last["total_bytes"] + NS * 12 + 8
    name, power = gpu_info()
    med = lambda v: float(np.median(v))  # noqa: E731
    print(json.dumps({
        "gpu": name, "power_limit": power, "n_streams": N_STREAMS, "capsules_per_push": CAPS, "max_nodes": MAX_NODES,
        "max_scans": MAX_SCANS, "messages_per_push": n_msgs,
        "d2h_bytes_padded_push_outputs": padded, "d2h_bytes_packed_messages": packed,
        "host_push_ms": med(host["push"]), "host_push_plus_laserscan_msgs_ms": med(host["push_msgs"]),
        "dev_push_ms": med(devt["push_dev"]), "dev_push_plus_laserscan_msgs_dev_ms": med(devt["push_dev_msgs"]),
        "rounds": {"host": host, "dev": devt},
    }))
    sess2.close()
    sess.close()
    ctx.close()


if __name__ == "__main__":
    main()
