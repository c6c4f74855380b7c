"""Session nodes (rpl_capsule_stream_nodes_dev) behind the push that published the scans; prints one JSON line.

Shapes: 512 dense-capsule streams (0x85), revolutions of about 3200 nodes:
  * the shape of bench.py --workload chain, 4096 capsules per stream and push, max_scans 56, at max_nodes 4096 and 8192;
  * a small push of 80 capsules per stream (a 25 ms receive period), max_nodes 4096, max_scans 4.
Per shape, CUDA-event time per push of push_dev alone, push_dev + nodes_dev ascended, and push_dev + nodes_dev passed
through (apply_ascend = 0), the three variants alternating in rounds within one run: medians and the rounds' ranges.
Also the bytes the host form copies device-to-host for one push (the packed buffers and the tables) against the padded
[n_streams * max_scans][max_nodes] node rows and statuses the stateless path would move, and the nodes call's
algorithmic traffic (8 B read + 8 B written per node, plus the tables).  Pushes continue the streams.  The GPU's name
and power limit are part of the output.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import feed  # noqa: E402
from bench_stream_msgs import gpu_info  # noqa: E402

N_STREAMS = 512
SHAPES = [("chain", 4096, 4096, 56), ("chain_8192", 4096, 8192, 56), ("small_push", 80, 4096, 4)]


def run_shape(R, torch, args, caps, max_nodes, max_scans):
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream()
    n_push = 2  # a pool of pushes replayed in turn: 16 distinct streams, repeated over the 512
    pool = feed(16, caps * n_push)
    d_pool = [torch.from_numpy(np.ascontiguousarray(pool[:, p * caps:(p + 1) * caps])).to(dev)
              .repeat(N_STREAMS // 16, 1, 1) for p in range(n_push)]
    d_cnt = torch.full((N_STREAMS,), caps, dtype=torch.int32, device=dev)
    NS = N_STREAMS * max_scans
    prm = R.scan_params(1, 0, 0, 1)
    ctx = R.Context(0, max_nodes, NS)
    r, it = torch.empty((NS, max_nodes), device=dev), torch.empty((NS, max_nodes), device=dev)
    bc, inc = torch.empty(NS, dtype=torch.int32, device=dev), torch.empty(NS, device=dev)
    sps = torch.empty(N_STREAMS, dtype=torch.int32, device=dev)
    cap = N_STREAMS * (caps * 40 + max_nodes) + NS  # every node decoded or carried, and the padding nodes
    d_nodes = torch.empty(cap, dtype=torch.int64, device=dev)
    d_off = torch.empty(NS, dtype=torch.int64, device=dev)
    d_cntn, d_stat = torch.empty(NS, dtype=torch.int32, device=dev), torch.empty(NS, dtype=torch.int32, device=dev)
    d_tot = torch.zeros(1, dtype=torch.int64, device=dev)
    sess = R.DenseStreamSession(ctx, N_STREAMS, caps, max_nodes, max_scans)
    k = [0]

    def run(variant):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(args.steps):
            sess.push_dev(d_pool[k[0] % n_push].data_ptr(), d_cnt.data_ptr(), prm, r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=st.cuda_stream)
            k[0] += 1
            if variant != "push_dev":
                sess.nodes_dev(d_nodes.data_ptr(), cap, d_off.data_ptr(), d_cntn.data_ptr(), d_stat.data_ptr(),
                               d_tot.data_ptr(), apply_ascend=variant == "push_dev_nodes_ascended",
                               stream=st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    variants = ("push_dev", "push_dev_nodes_ascended", "push_dev_nodes_passed")
    for _ in range(args.warmup):
        for v in variants:
            run(v)
    ms = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            ms[v].append(run(v))
    total = int(d_tot.cpu().numpy()[0])
    assert 0 < total <= cap, "the buffers of the last push must fit"
    n_bufs = int((d_cntn.cpu().numpy() > 0).sum())
    sess.close()
    ctx.close()
    res = {"capsules_per_push": caps, "max_nodes": max_nodes, "max_scans": max_scans, "buffers_last_push": n_bufs,
           "nodes_last_push": total,
           "d2h_bytes_host_form": total * 8 + NS * 16 + 8,
           "d2h_bytes_padded_rows": NS * max_nodes * 8 + NS * 4,
           "algorithmic_bytes_nodes_call": total * 16 + NS * (8 + 8 + 4 + 4 + 8)}
    for v in variants:
        res[v + "_ms"] = {"median": float(np.median(ms[v])), "min": min(ms[v]), "max": max(ms[v])}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed pushes per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    if not torch.cuda.is_available():
        sys.exit("bench_stream_nodes.py needs a CUDA device (an H100): there is nothing to time without one")
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "n_streams": N_STREAMS, "steps": args.steps, "rounds": args.rounds}
    for label, caps, max_nodes, max_scans in SHAPES:
        out[label] = run_shape(R, torch, args, caps, max_nodes, max_scans)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
