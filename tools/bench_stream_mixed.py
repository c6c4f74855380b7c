"""What serving several answer types from one byte session (rpl_capsule_stream_create_bytes_mixed) costs a device push;
prints one JSON line.

Shape: the chain shape of bench.py in bytes, 512 streams x 344064 bytes per push (4096 dense capsules' worth), split
across the six answer types (stream s of type 0x81 + s % 6: about 85 streams each), max_nodes 4096, max_scans 56.
push_bytes_dev is timed with CUDA events, in rounds that alternate the two forms:
  mixed   one mixed session of the 512 streams: per chunk the framer, decoder and assembler once per type, the scan
          kernels once;
  single  the same streams as six single-type byte sessions, one push each.
Every push replays each stream's same bytes, so a stream continues with one angular jump per push (and, where the
push is not a whole number of frames, a frame completed across it).  The medians over the rounds are reported, with the
GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dense_stream import FORMATS, feed, feed_format, feed_normal  # noqa: E402
from bench_stream_lidars import gpu_info  # noqa: E402

N_STREAMS, PUSH_BYTES, MAX_NODES, MAX_SCANS = 512, 4096 * 84, 4096, 56
TYPES = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]


def stream_bytes():
    """[N_STREAMS, PUSH_BYTES]: stream s carries answer type TYPES[s % 6]"""
    out = np.empty((N_STREAMS, PUSH_BYTES), np.uint8)
    for k, t in enumerate(TYPES):
        rows = np.arange(k, N_STREAMS, 6)
        if t == 0x81:
            out[rows] = feed_normal(len(rows), PUSH_BYTES, seed=k + 1)
            continue
        if t == 0x85:
            caps = feed(len(rows), PUSH_BYTES // 84, seed=k + 1)
        else:
            caps = feed_format(t, len(rows), -(-PUSH_BYTES // FORMATS[t][0]), seed=k + 1)
        out[rows] = caps.reshape(len(rows), -1)[:, :PUSH_BYTES]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed pushes per form and round")
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
    b = stream_bytes()
    types = np.array([TYPES[s % 6] for s in range(N_STREAMS)], np.uint32)
    d_b = torch.from_numpy(b).to(dev)
    d_cnt = torch.full((N_STREAMS,), PUSH_BYTES, dtype=torch.int32, device=dev)
    order = np.argsort(types, kind="stable")  # the single-type sessions' streams, back to back
    d_sorted = d_b[torch.from_numpy(order).to(dev)].contiguous()
    NS = N_STREAMS * MAX_SCANS
    r = torch.empty((NS, MAX_NODES), device=dev)
    it = torch.empty((NS, MAX_NODES), device=dev)
    bc = torch.empty(NS, dtype=torch.int32, device=dev)
    inc = torch.empty(NS, device=dev)
    sps = torch.empty(N_STREAMS, dtype=torch.int32, device=dev)
    ctx = R.Context(0, MAX_NODES, NS)
    params = R.scan_params(1, 0, 0, 1)

    mixed = R.MixedByteStreamSession(ctx, types, PUSH_BYTES, MAX_NODES, MAX_SCANS)
    singles, first = [], 0
    for t in TYPES:
        n = int((types == t).sum())
        singles.append((R.CapsuleByteStreamSession(ctx, t, n, PUSH_BYTES, MAX_NODES, MAX_SCANS), first, n))
        first += n

    def push(sess, d_in, s0, n):
        o = s0 * MAX_SCANS
        sess.push_dev(d_in[s0:].data_ptr(), d_cnt.data_ptr(), params, r[o:].data_ptr(), it[o:].data_ptr(),
                      bc[o:].data_ptr(), inc[o:].data_ptr(), sps[s0:].data_ptr(), stream=st.cuda_stream)

    def push_singles():
        for sess, s0, n in singles:
            push(sess, d_sorted, s0, n)

    steps = {"mixed": lambda: push(mixed, d_b, 0, N_STREAMS), "single": push_singles}

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
    scans = {}
    for k, fn in steps.items():  # scans one push publishes, per form
        fn()
        torch.cuda.synchronize()
        scans[k] = int(sps.sum().item())
    rounds = {k: [] for k in steps}
    for _ in range(args.rounds):
        for k, fn in steps.items():
            rounds[k].append(timed(fn, args.steps))
    med = {k: float(np.median(v)) for k, v in rounds.items()}
    print(json.dumps({
        "gpu": name, "power_limit": power, "n_streams": N_STREAMS, "bytes_per_push": PUSH_BYTES,
        "max_nodes": MAX_NODES, "max_scans": MAX_SCANS, "scans_per_push": scans,
        "push_bytes_dev_ms": {f"{k}_median": v for k, v in med.items()}, "mixed_over_single": med["mixed"] / med["single"],
        "rounds_ms": rounds,
    }))
    mixed.close()
    for sess, _, _ in singles:
        sess.close()
    ctx.close()


if __name__ == "__main__":
    main()
