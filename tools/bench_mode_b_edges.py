"""Where the LaserScan Mode B headline step spends the time outside the cluster kernel's steady state; one JSON line.

The shape of bench.py's headline: 4096 scans x 32768 nodes, Mode B, device-resident, on a non-default stream, one
rpl_scan_batch_dev call per step.  Reported:
  * CUDA-event step time with the context's profiling off and on, alternating in rounds (medians and ranges);
  * the fast and general kernel times rpl_ctx_profile_read returns for the profiled rounds;
  * from torch.profiler traces of --trace-steps steps (one with profiling off, one on, written under --out): the
    median duration of every device activity of a step (memset, cluster kernel, general kernel) and the median gap
    between each consecutive pair of them, the gap between steps included;
  * the GPU's name, power limit and SM clocks, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (x.strip() for x in out.split(","))))
    except Exception:  # noqa: BLE001
        return {"name": "unknown"}


def kind(ev):
    name = ev.get("name", "")
    if ev.get("cat") == "gpu_memset":
        return "memset"
    if "scan_tma_cluster_kernel" in name:
        return "cluster"
    if "scan_general_kernel" in name:
        return "general"
    return name[:48]


def trace_summary(path):
    """median duration per activity kind and median gap per consecutive pair of kinds (microseconds)"""
    with open(path) as f:
        evs = [e for e in json.load(f)["traceEvents"]
               if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    evs.sort(key=lambda e: e["ts"])
    dur, gap = {}, {}
    for i, e in enumerate(evs):
        dur.setdefault(kind(e), []).append(e["dur"])
        if i:
            p = evs[i - 1]
            gap.setdefault(f"{kind(p)}->{kind(e)}", []).append(e["ts"] - (p["ts"] + p["dur"]))
    med = lambda d: {k: round(statistics.median(v), 3) for k, v in d.items()}  # noqa: E731
    return {"activities": len(evs), "duration_us": med(dur), "gap_us": med(gap)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=4096)
    ap.add_argument("--nodes", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=200, help="timed steps per round and setting")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--trace-steps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "mode_b_edges"),
                    help="directory for the profiler traces")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import rplidar_ros2_driver_b200 as R

    if not torch.cuda.is_available():
        raise SystemExit("bench_mode_b_edges.py needs a CUDA device")
    S, N = args.scans, args.nodes
    dev = torch.device("cuda", 0)
    ctx = R.Context(0, N, S)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    sp = st.cuda_stream
    nodes = torch.empty((S, N, 8), dtype=torch.uint8, device=dev)
    counts = torch.empty(S, dtype=torch.int32, device=dev)
    ranges = torch.empty((S, N), dtype=torch.float32, device=dev)
    intens = torch.empty((S, N), dtype=torch.float32, device=dev)
    small = [torch.empty(S, dtype=torch.int32, device=dev) for _ in range(4)]
    ctx.synth_batch_dev(0, S, N, N, 0, nodes.data_ptr(), counts.data_ptr(), stream=sp)
    params = R.scan_params(0, 0, 0, 1)

    def step():
        ctx.scan_batch_dev(nodes.data_ptr(), counts.data_ptr(), S, N, params, ranges=ranges.data_ptr(),
                           intensities=intens.data_ptr(), beam_counts=small[0].data_ptr(),
                           angle_increment=small[1].data_ptr(), status=small[2].data_ptr(), path=small[3].data_ptr(),
                           stream=sp)

    def timed(prof_on, k):
        ctx.profile(prof_on)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(k):
            step()
        e1.record(st)
        torch.cuda.synchronize()
        pr = ctx.profile_read()
        ctx.profile(False)
        return e0.elapsed_time(e1) / k, pr

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    ctx.profile_read()
    step_ms = {"profile_off": [], "profile_on": []}
    fast_ms, general_ms, launches = [], [], None
    for _ in range(args.rounds):
        step_ms["profile_off"].append(timed(False, args.steps)[0])
        ms, pr = timed(True, args.steps)
        step_ms["profile_on"].append(ms)
        fast_ms.append(pr[0] / max(pr[1], 1))
        general_ms.append(pr[2] / max(pr[3], 1))
        launches = (pr[1], pr[3])
    fast_on = int((small[3] == 0).sum().item())

    os.makedirs(args.out, exist_ok=True)
    traces = {}
    for prof_on in (False, True):
        ctx.profile(prof_on)
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(args.trace_steps):
                step()
            torch.cuda.synchronize()
        ctx.profile(False)
        ctx.profile_read()
        path = os.path.join(args.out, f"trace_profile_{'on' if prof_on else 'off'}.pt.trace.json")
        p.export_chrome_trace(path)
        traces["profile_on" if prof_on else "profile_off"] = trace_summary(path)

    rng = lambda v: [round(min(v), 5), round(max(v), 5)]  # noqa: E731
    print(json.dumps({
        "shape": {"scans": S, "nodes": N, "mode": "B"}, "gpu": gpu_info(),
        "lib": os.environ.get("RPL_B200_LIB") or "in-tree",
        "step_ms": {k: {"median": round(statistics.median(v), 5), "range": rng(v)} for k, v in step_ms.items()},
        "profile_read": {"fast_ms": round(statistics.median(fast_ms), 5),
                         "general_ms": round(statistics.median(general_ms), 5),
                         "launches_per_round": {"fast": launches[0], "general": launches[1]}},
        "scans_on_fast_kernel": fast_on, "traces": traces}), flush=True)


if __name__ == "__main__":
    main()
