"""Stream session timings on the GPU; prints one JSON line.

With --format 0x85 (the default), the dense stream session (rpl_capsule_stream_* on 0x85):

  * per-push latency of push (host buffers, synchronous) and push_dev (device buffers, CUDA events on a torch stream)
    for 512 streams x {8, 80, 800} capsules per push: a live aggregator's receive periods of ~2.5 ms, ~25 ms, ~250 ms
    at 10 Hz, 80 capsules per revolution;
  * device-resident throughput of push_dev on the shape of bench.py --workload chain (512 streams x 4096 capsules,
    max_nodes 4096, max_scans 56), in nodes decoded per second: the figure to set next to that workload's.

With --format 0x82 / 0x83 / 0x84 / 0x86, the capsule stream session (rpl_capsule_stream_*) of that format against the
stateless device path on the same capsules (rpl_decode_capsules_batch_dev -> rpl_assemble_scan_views_dev ->
rpl_scan_views_dev): a chain-like shape of 512 streams x about 163840 nodes per push (the chain's 4096 dense capsules
x 40), revolutions of about 3200 nodes, max_nodes 4096, max_scans 56.

With --format 0x81, the standard-node stream session (rpl_capsule_stream_*_bytes on 0x81) on raw byte streams: the same
comparison against the stateless device path (rpl_decode_normal_batch_dev -> rpl_assemble_scan_views_dev ->
rpl_scan_views_dev) on 512 streams x 163840 five-byte records per push, revolutions of 3200 records, max_nodes 4096,
max_scans 56; and the per-push latency of push and push_dev for 512 streams x {100, 1000, 10000} bytes (at 115200 baud a
standard-mode lidar delivers about 11500 bytes per second).

With --stamped (any --format), stamped pushes (rpl_*_stream_push_ts_dev, receive times in, scan-begin stamps out)
against unstamped ones on the same data and shapes: the chain shape above for 0x85, the comparison shapes above for the
other formats; two sessions, timed in alternating rounds in one run.  Also the host push of a 25 ms receive period
(512 streams x 80 dense capsules, or the format's equivalent), stamped and unstamped, with the bytes each copies.

With --bytes (--format 0x82..0x86), byte pushes (rpl_capsule_stream_push_bytes_dev: raw bytes framed on the device,
the search for the sync bytes carried across pushes) against framed pushes (rpl_capsule_stream_push_dev) of the same
clean stream: the chain shape for 0x85 (512 streams x 4096 capsules), the comparison shapes above for the other formats,
and small pushes of 512 streams x about 2 KB (a 20 ms receive period at 1 Mbaud).  Two byte sessions: one pushed whole
capsules (every push starts on a frame), one pushed a byte count that is no multiple of the frame size, so most pushes
begin with held bytes and the stream sits off the word grid; three sessions timed in alternating rounds in one run.

With --cloud, the session clouds (rpl_capsule_stream_cloud_dev): push_dev alone against push_dev + cloud_dev with the
window only, 5 cm voxels, and SOR k=8 + 5 cm voxels, the last two fused (flags 0) and as separate passes
(RPL_CLOUD_NO_FUSED), at max_nodes 4096 and 8192 (at 8192 the fused kernel's shared memory is sized for 4096 nodes and
longer revolutions go to the general kernel), on the chain shape of 0x85 and the comparison shape of 0x84 (or of
--format): 512 streams, revolutions of about 3200 nodes; all timed in alternating rounds in one run.

Each push continues the stream where the previous one ended (the capsules of a push follow on in angle), so the carry
and the held capsule are exercised as in a live feed.  The GPU's name and power limit are part of the output.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import wire_dense_capsules, wire_seal_capsules  # noqa: E402

# per format: bytes and nodes per capsule, capsules per push (about 163840 nodes), capsules per revolution (~3200 nodes)
FORMATS = {0x82: (84, 32, 5120, 100.0), 0x83: (781, 96, 1707, 100.0 / 3), 0x84: (132, 96, 1707, 100.0 / 3),
           0x86: (170, 64, 2560, 50.0)}


def feed(n_streams, n_caps, seed=1):
    """[n_streams, n_caps, 84]: 80 capsules per revolution, 5 % zero distances, every stream at its own angle"""
    rng = np.random.default_rng(seed)
    out = np.empty((n_streams, n_caps, 84), np.uint8)
    for s in range(n_streams):
        ang = (rng.uniform(0, 360) + np.arange(n_caps) * 4.5 + rng.normal(0, 0.03, n_caps)) % 360.0
        q6 = np.round(ang * 64).astype(np.uint32) % (360 * 64)
        dist = rng.integers(1, 40000, (n_caps, 40))
        dist[rng.random((n_caps, 40)) < 0.05] = 0
        out[s] = wire_dense_capsules(q6, np.zeros(n_caps, bool), dist)
    return out


def feed_format(fmt, n_streams, n_caps, seed=1):
    """[n_streams, n_caps, capsule bytes] of format `fmt`: random payloads, start angles (HQ: node angles and scan-start
    flags) rising through revolutions of about 3200 nodes, every stream at its own angle"""
    cb, per, _, cpr = FORMATS[fmt]
    rng = np.random.default_rng(seed)
    out = np.empty((n_streams, n_caps, cb), np.uint8)
    for s in range(n_streams):
        payload = rng.integers(0, 256, (n_caps, cb), dtype=np.uint8)
        if fmt == 0x83:
            # nodes: angle_z_q14 u16 | dist_mm_q2 u32 | quality u8 | flag u8 (scan start on each revolution's first)
            m, npr = n_caps * per, int(round(cpr * per))
            pos = (np.arange(m) + int(rng.integers(0, npr))) % npr
            dist = rng.integers(4, 160000, m).astype(np.uint32)
            w = np.empty((m, 2), np.uint32)
            w[:, 0] = (pos * 65536 // npr).astype(np.uint32) | ((dist & 0xFFFF) << 16)
            w[:, 1] = (dist >> 16) | (rng.integers(0, 256, m).astype(np.uint32) << 16) | \
                (np.where(pos == 0, 1, 2).astype(np.uint32) << 24)
            payload[:, 9:9 + 8 * per] = w.view(np.uint8).reshape(n_caps, 8 * per)
            out[s] = wire_seal_capsules(fmt, payload)
        else:
            ang = (rng.uniform(0, 360) + np.arange(n_caps) * 360.0 / cpr + rng.normal(0, 0.03, n_caps)) % 360.0
            q6 = np.round(ang * 64).astype(np.uint32) % (360 * 64)
            out[s] = wire_seal_capsules(fmt, payload, q6, np.zeros(n_caps, bool))
    return out


def feed_normal(n_streams, n_bytes, seed=1):
    """[n_streams, n_bytes] of 0x81 records: angles rising through revolutions of 3200 records whose first carries the
    sync bit, 5 % zero distances, every stream at its own angle; a push may end inside a record"""
    rng = np.random.default_rng(seed)
    n_rec = (n_bytes + 4) // 5
    out = np.empty((n_streams, n_rec * 5), np.uint8)
    for s in range(n_streams):
        pos = (np.arange(n_rec) + int(rng.integers(0, 3200))) % 3200
        start = (pos == 0).astype(np.uint8)
        rec = out[s].reshape(n_rec, 5)
        rec[:, 0] = (rng.integers(0, 64, n_rec).astype(np.uint8) << 2) | ((1 - start) << 1) | start
        w = ((pos * (360 * 64) // 3200) << 1) | 1
        rec[:, 1], rec[:, 2] = w & 0xFF, w >> 8
        dist = rng.integers(4, 65536, n_rec)
        dist[rng.random(n_rec) < 0.05] = 0
        rec[:, 3], rec[:, 4] = dist & 0xFF, dist >> 8
    return out[:, :n_bytes]


def compare_normal(R, torch, steps):
    """ms per push of the standard-node session's push_dev and of the stateless device path, on the same bytes"""
    n_streams, n_bytes, max_nodes, max_scans = 512, 163840 * 5, 4096, 56
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    feed_ = feed_normal(16, 2 * n_bytes, seed=7)
    NS, stride_nodes = n_streams * max_scans, n_bytes // 5
    res = {"format": "0x81", "streams": n_streams, "bytes_per_push": n_bytes, "nodes_per_push_per_stream": stride_nodes,
           "max_nodes": max_nodes, "max_scans": max_scans}
    with torch.cuda.stream(stream):
        halves = [torch.from_numpy(np.ascontiguousarray(feed_[:, h * n_bytes:(h + 1) * n_bytes])).to(dev)
                  .repeat(n_streams // 16, 1) for h in (0, 1)]
        d_cnt = torch.full((n_streams,), n_bytes, dtype=torch.int32, device=dev)
        r = torch.empty((NS, max_nodes), device=dev)
        it = torch.empty((NS, max_nodes), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        nodes = torch.empty(n_streams * stride_nodes, dtype=torch.int64, device=dev)
        node_counts = torch.empty(n_streams, dtype=torch.int32, device=dev)
        views = torch.empty(NS, dtype=torch.int64, device=dev)
        scan_len = torch.empty(NS, dtype=torch.int32, device=dev)
    cs = stream.cuda_stream

    def stateless(t):
        ctx.decode_normal_batch_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), n_streams, n_bytes, nodes.data_ptr(),
                                    node_counts.data_ptr(), stream=cs)
        ctx.assemble_scan_views_dev(nodes.data_ptr(), node_counts.data_ptr(), n_streams, stride_nodes, max_nodes,
                                    max_scans, views.data_ptr(), scan_len.data_ptr(), sps.data_ptr(), stream=cs)
        ctx.scan_views_dev(nodes.data_ptr(), n_streams * stride_nodes, views.data_ptr(), NS, max_nodes, params,
                           ranges=r.data_ptr(), intensities=it.data_ptr(), beam_counts=bc.data_ptr(),
                           angle_increment=inc.data_ptr(), stream=cs)

    res["stateless_ms_per_push"] = timed(torch, stream, stateless, steps)
    res["stateless_scans_per_push"] = int(sps.cpu().sum())
    with R.NormalStreamSession(ctx, n_streams, n_bytes, max_nodes, max_scans) as sess:
        def push(t):
            sess.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=cs)

        res["push_dev_ms_per_push"] = timed(torch, stream, push, steps)
        res["push_dev_scans_per_push"] = int(sps.cpu().sum())
    res["push_dev_gnodes_per_s"] = n_streams * stride_nodes / (res["push_dev_ms_per_push"] * 1e-3) / 1e9
    res["session_over_stateless"] = res["push_dev_ms_per_push"] / res["stateless_ms_per_push"] - 1.0
    ctx.close()
    return res


def normal_latency(R, torch, pushes):
    """per-push latency of the standard-node session for 512 streams x {100, 1000, 10000} bytes per push"""
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    n_streams, max_nodes, max_scans = 512, 4096, 16
    rep = n_streams // 16
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    rows = []
    for per in (100, 1000, 10000):
        feed_ = feed_normal(16, per * (pushes + 4), seed=per)
        counts = np.full(n_streams, per, np.uint32)
        row = {"streams": n_streams, "bytes_per_push": per}
        with R.NormalStreamSession(ctx, n_streams, per, max_nodes, max_scans) as sess:
            pin = torch.empty((n_streams, per), dtype=torch.uint8).pin_memory().numpy()
            out = pinned_outputs(torch, n_streams, max_nodes, max_scans)
            ts = []
            for t in range(pushes + 4):
                pin[:] = np.tile(feed_[:, t * per:(t + 1) * per], (rep, 1))
                t0 = time.perf_counter()
                sess.push(pin, counts, params, out=out)
                ts.append(time.perf_counter() - t0)
            ts = np.array(ts[4:]) * 1e3
            row["push_ms_median"], row["push_ms_p90"] = float(np.median(ts)), float(np.percentile(ts, 90))
        with R.NormalStreamSession(ctx, n_streams, per, max_nodes, max_scans) as sess, torch.cuda.stream(stream):
            d_feed = torch.from_numpy(feed_).to(dev)
            d_cnt = torch.full((n_streams,), per, dtype=torch.int32, device=dev)
            NS = n_streams * max_scans
            r = torch.empty((NS, max_nodes), device=dev)
            it = torch.empty((NS, max_nodes), device=dev)
            bc = torch.zeros(NS, dtype=torch.int32, device=dev)
            inc = torch.zeros(NS, device=dev)
            sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(pushes + 4)]
            for t in range(pushes + 4):
                piece = d_feed[:, t * per:(t + 1) * per].repeat(rep, 1)
                evs[t][0].record(stream)
                sess.push_dev(piece.data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                              inc.data_ptr(), sps.data_ptr(), stream=stream.cuda_stream)
                evs[t][1].record(stream)
            stream.synchronize()
            ms = np.array([a.elapsed_time(b) for a, b in evs[4:]])
            row["push_dev_ms_median"], row["push_dev_ms_p90"] = float(np.median(ms)), float(np.percentile(ms, 90))
        rows.append(row)
    ctx.close()
    return rows


def pinned_outputs(torch, n_streams, max_nodes, max_scans):
    """the output dict of push in pinned host memory, as an aggregator would keep it"""
    out = {k: torch.zeros(shape, dtype=dt).pin_memory().numpy() for k, shape, dt in (
        ("ranges", (n_streams * max_scans, max_nodes), torch.float32),
        ("intensities", (n_streams * max_scans, max_nodes), torch.float32),
        ("beam_counts", (n_streams * max_scans,), torch.int32), ("angle_increment", (n_streams * max_scans,), torch.float32),
        ("scans_per_stream", (n_streams,), torch.int32))}
    out["beam_counts"] = out["beam_counts"].view(np.uint32)
    out["scans_per_stream"] = out["scans_per_stream"].view(np.uint32)
    return out


def timed(torch, stream, fn, steps):
    """ms per call of fn(t) on `stream`, CUDA events around `steps` calls after 4 warm-up calls"""
    for t in range(4):
        fn(t)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for t in range(steps):
        fn(t)
    e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1) / steps


def compare_stateless(R, torch, fmt, steps):
    """ms per push of the session's push_dev and of the stateless device path, on the same capsules"""
    _, per, n_caps, _ = FORMATS[fmt]
    n_streams, max_nodes, max_scans = 512, 4096, 56
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    caps = feed_format(fmt, 16, n_caps * 2, seed=7)
    NS, stride_nodes = n_streams * max_scans, n_caps * per
    res = {"format": hex(fmt), "streams": n_streams, "capsules_per_push": n_caps, "nodes_per_push_per_stream": stride_nodes,
           "max_nodes": max_nodes, "max_scans": max_scans}
    with torch.cuda.stream(stream):
        halves = [torch.from_numpy(np.tile(caps[:, h * n_caps:(h + 1) * n_caps], (n_streams // 16, 1, 1))).to(dev)
                  for h in (0, 1)]
        d_cnt = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
        r = torch.empty((NS, max_nodes), device=dev)
        it = torch.empty((NS, max_nodes), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        nodes = torch.empty(n_streams * stride_nodes, dtype=torch.int64, device=dev)
        node_counts = torch.empty(n_streams, dtype=torch.int32, device=dev)
        status = torch.empty(n_streams * n_caps, dtype=torch.int32, device=dev)
        offs = torch.empty(n_streams * n_caps, dtype=torch.int32, device=dev)
        views = torch.empty(NS, dtype=torch.int64, device=dev)
        scan_len = torch.empty(NS, dtype=torch.int32, device=dev)
    cs = stream.cuda_stream

    def stateless(t):
        ctx.decode_capsules_batch_dev(fmt, halves[t % 2].data_ptr(), d_cnt.data_ptr(), n_streams, n_caps, 31,
                                      nodes.data_ptr(), node_counts.data_ptr(), capsule_status=status.data_ptr(),
                                      capsule_node_offset=offs.data_ptr(), stream=cs)
        ctx.assemble_scan_views_dev(nodes.data_ptr(), node_counts.data_ptr(), n_streams, stride_nodes, max_nodes,
                                    max_scans, views.data_ptr(), scan_len.data_ptr(), sps.data_ptr(),
                                    capsule_status=status.data_ptr(), capsule_node_offset=offs.data_ptr(),
                                    capsule_counts=d_cnt.data_ptr(), stride_capsules=n_caps, stream=cs)
        ctx.scan_views_dev(nodes.data_ptr(), n_streams * stride_nodes, views.data_ptr(), NS, max_nodes, params,
                           ranges=r.data_ptr(), intensities=it.data_ptr(), beam_counts=bc.data_ptr(),
                           angle_increment=inc.data_ptr(), stream=cs)

    res["stateless_ms_per_push"] = timed(torch, stream, stateless, steps)
    res["stateless_scans_per_push"] = int(sps.cpu().sum())
    with R.CapsuleStreamSession(ctx, fmt, n_streams, n_caps, max_nodes, max_scans) as sess:
        def push(t):
            sess.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=cs)

        res["push_dev_ms_per_push"] = timed(torch, stream, push, steps)
        res["push_dev_scans_per_push"] = int(sps.cpu().sum())
    res["push_dev_gnodes_per_s"] = n_streams * stride_nodes / (res["push_dev_ms_per_push"] * 1e-3) / 1e9
    res["session_over_stateless"] = res["push_dev_ms_per_push"] / res["stateless_ms_per_push"] - 1.0
    ctx.close()
    return res


def compare_stamped(R, torch, fmt, steps, rounds):
    """ms per push_dev of a stamped and an unstamped session on the same data, alternating rounds of `steps` pushes;
    and ms per host push of a 25 ms receive period, stamped and unstamped"""
    n_streams, max_nodes, max_scans = 512, 4096, 56
    if fmt == 0x81:
        cb, n_units, host_units = 1, 163840 * 5, 1000
        data = feed_normal(16, 2 * n_units, seed=7)
    elif fmt == 0x85:
        cb, n_units, host_units = 84, 4096, 80
        data = feed(16, 2 * n_units, seed=7)
    else:
        cb, _, n_units, cpr = FORMATS[fmt]
        host_units = int(round(cpr))  # one revolution, as the dense session's 80 capsules
        data = feed_format(fmt, 16, 2 * n_units, seed=7)
    chunk_bytes = 64  # 0x81: one receive time per 64 bytes
    n_rx = -(-n_units // chunk_bytes) if fmt == 0x81 else n_units
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    timing = R.Timing(31, 0, 0, 0)
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    NS = n_streams * max_scans
    reps = (n_streams // 16,) + (1,) * (data.ndim - 1)
    with torch.cuda.stream(stream):
        halves = [torch.from_numpy(np.ascontiguousarray(np.tile(data[:, h * n_units:(h + 1) * n_units], reps))).to(dev)
                  for h in (0, 1)]
        d_cnt = torch.full((n_streams,), n_units, dtype=torch.int32, device=dev)
        rx = [(torch.arange(n_streams * n_rx, device=dev, dtype=torch.int64) * 10 + 10_000_000 + h).reshape(n_streams, n_rx)
              for h in (0, 1)]
        r = torch.empty((NS, max_nodes), device=dev)
        it = torch.empty((NS, max_nodes), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
        ts = torch.zeros(NS, dtype=torch.int64, device=dev)
    cs = stream.cuda_stream

    def session(stride):
        if fmt == 0x81:
            return R.NormalStreamSession(ctx, n_streams, stride, max_nodes, max_scans)
        return R.CapsuleStreamSession(ctx, fmt, n_streams, stride, max_nodes, max_scans)

    def stamp_kw(rx_ptr, ts_ptr):
        if fmt == 0x81:
            return dict(chunk_bytes=chunk_bytes, chunk_rx_us=rx_ptr, timing=timing, scan_begin_ts_us=ts_ptr)
        return dict(rx_us=rx_ptr, timing=timing, scan_begin_ts_us=ts_ptr)

    res = {"format": hex(fmt), "streams": n_streams, "units_per_push": n_units, "unit_bytes": cb, "max_nodes": max_nodes,
           "max_scans": max_scans, "steps": steps, "rounds": rounds, "plain_ms": [], "stamped_ms": []}
    with session(n_units) as plain, session(n_units) as stamped:
        def push_plain(t):
            plain.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                           bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=cs)

        def push_stamped(t):
            stamped.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                             bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=cs,
                             **stamp_kw(rx[t % 2].data_ptr(), ts.data_ptr()))

        for _ in range(rounds):
            res["plain_ms"].append(timed(torch, stream, push_plain, steps))
            res["stamped_ms"].append(timed(torch, stream, push_stamped, steps))
        res["scans_per_push"] = int(sps.cpu().sum())
    res["plain_ms_median"] = float(np.median(res["plain_ms"]))
    res["stamped_ms_median"] = float(np.median(res["stamped_ms"]))
    res["stamped_over_plain"] = res["stamped_ms_median"] / res["plain_ms_median"] - 1.0
    # host pushes of one receive period: input bytes and the receive times' extra bytes, copied per push
    h_data = np.ascontiguousarray(np.tile(data[:, :host_units], reps))
    h_cnt = np.full(n_streams, host_units, np.uint32)
    h_rx_n = -(-host_units // chunk_bytes) if fmt == 0x81 else host_units
    h_rx = np.arange(n_streams * h_rx_n, dtype=np.uint64).reshape(n_streams, h_rx_n) + 10_000_000
    out = pinned_outputs(torch, n_streams, max_nodes, max_scans)
    out["scan_begin_ts_us"] = torch.zeros(NS, dtype=torch.int64).pin_memory().numpy().view(np.uint64)
    host = {"units_per_push": host_units, "input_bytes": int(h_data.nbytes), "rx_bytes": int(h_rx.nbytes),
            "plain_ms": [], "stamped_ms": []}
    with session(host_units) as plain, session(host_units) as stamped:
        kw = dict(chunk_bytes=chunk_bytes, chunk_rx_us=h_rx, timing=timing) if fmt == 0x81 else \
            dict(rx_us=h_rx, timing=timing)
        for t in range(4 + 2 * steps):
            for sess, extra, key in ((plain, {}, "plain_ms"), (stamped, kw, "stamped_ms")):
                t0 = time.perf_counter()
                sess.push(h_data, h_cnt, params, out=out, **extra)
                if t >= 4:
                    host[key].append((time.perf_counter() - t0) * 1e3)
    host["plain_ms_median"] = float(np.median(host.pop("plain_ms")))
    host["stamped_ms_median"] = float(np.median(host.pop("stamped_ms")))
    host["stamped_over_plain"] = host["stamped_ms_median"] / host["plain_ms_median"] - 1.0
    res["host_push"] = host
    ctx.close()
    return res


def byte_windows(torch, dev, caps, n_streams, P):
    """caps [16, M, cb] read as a ring of M * cb bytes per stream (a whole number of pushes of P bytes): the device
    buffers [n_streams, P] of the pushes that walk once around it, tiled over n_streams"""
    flat = caps.reshape(caps.shape[0], -1)
    W = flat.shape[1] // P
    assert W * P == flat.shape[1]
    return [torch.from_numpy(np.ascontiguousarray(np.tile(flat[:, w * P:(w + 1) * P], (n_streams // 16, 1)))).to(dev)
            for w in range(W)]


def compare_bytes(R, torch, fmt, steps, rounds, small):
    """ms per push_dev of a framed session, a byte session pushed whole capsules and a byte session pushed a byte count
    off the frame grid, on clean streams of `fmt`, alternating rounds of `steps` pushes"""
    n_streams, max_nodes, max_scans = 512, 4096, 56
    if fmt == 0x85:
        cb, n_units = 84, 4096

        def gen(m, seed):
            return feed(16, m, seed)
    else:
        cb, _, n_units, _ = FORMATS[fmt]

        def gen(m, seed):
            return feed_format(fmt, 16, m, seed)
    if small:  # about 2 KB per push: framed pushes carry the whole capsules in it, byte pushes 2048 bytes
        n_units, P = max(1, 2048 // cb), 2048
        W = cb // math.gcd(cb, P)
    else:  # the byte count of W pushes is a whole number of frames: W - 1 of W pushes begin with held bytes
        W = min(w for w in range(3, cb + 1) if cb % w == 0)
        P = n_units * cb - cb // W
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    NS = n_streams * max_scans
    data = gen(2 * n_units, 7)
    ring = gen(W * P // cb, 8)
    with torch.cuda.stream(stream):
        halves = [torch.from_numpy(np.ascontiguousarray(np.tile(data[:, h * n_units:(h + 1) * n_units],
                                                                (n_streams // 16, 1, 1)))).to(dev) for h in (0, 1)]
        windows = byte_windows(torch, dev, ring, n_streams, P)
        cnt_caps = torch.full((n_streams,), n_units, dtype=torch.int32, device=dev)
        cnt_al = torch.full((n_streams,), n_units * cb, dtype=torch.int32, device=dev)
        cnt_mis = torch.full((n_streams,), P, dtype=torch.int32, device=dev)
        r = torch.empty((NS, max_nodes), device=dev)
        it = torch.empty((NS, max_nodes), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    cs = stream.cuda_stream
    outs = (r.data_ptr(), it.data_ptr(), bc.data_ptr(), inc.data_ptr(), sps.data_ptr())
    res = {"format": hex(fmt), "streams": n_streams, "capsules_per_framed_push": n_units,
           "bytes_per_aligned_push": n_units * cb, "bytes_per_offgrid_push": P, "offgrid_pushes_per_cycle": W,
           "max_nodes": max_nodes, "max_scans": max_scans, "steps": steps, "rounds": rounds,
           "framed_ms": [], "bytes_aligned_ms": [], "bytes_offgrid_ms": []}
    scans = {}
    with R.CapsuleStreamSession(ctx, fmt, n_streams, n_units, max_nodes, max_scans) as framed, \
            R.CapsuleByteStreamSession(ctx, fmt, n_streams, n_units * cb, max_nodes, max_scans) as aligned, \
            R.CapsuleByteStreamSession(ctx, fmt, n_streams, P, max_nodes, max_scans) as offgrid:
        def push_framed(t):
            framed.push_dev(halves[t % 2].data_ptr(), cnt_caps.data_ptr(), params, *outs, stream=cs)

        def push_aligned(t):
            aligned.push_dev(halves[t % 2].data_ptr(), cnt_al.data_ptr(), params, *outs, stream=cs)

        def push_offgrid(t):
            offgrid.push_dev(windows[t % W].data_ptr(), cnt_mis.data_ptr(), params, *outs, stream=cs)

        for _ in range(rounds):
            for key, fn in (("framed_ms", push_framed), ("bytes_aligned_ms", push_aligned),
                            ("bytes_offgrid_ms", push_offgrid)):
                res[key].append(timed(torch, stream, fn, steps))
                scans[key] = int(sps.cpu().sum())
        res["held_bytes_offgrid"] = sorted(set(offgrid.state()[2].tolist()))
    res["scans_per_push"] = scans
    for key in ("framed_ms", "bytes_aligned_ms", "bytes_offgrid_ms"):
        res[key + "_median"] = float(np.median(res[key]))
    res["aligned_over_framed"] = res["bytes_aligned_ms_median"] / res["framed_ms_median"] - 1.0
    res["offgrid_over_framed"] = res["bytes_offgrid_ms_median"] / res["framed_ms_median"] - 1.0
    ctx.close()
    return res


def compare_cloud(R, torch, fmt, steps, rounds):
    """ms per push_dev alone and per push_dev + cloud_dev (window only; 5 cm voxels; SOR k=8 + 5 cm voxels; fused and
    RPL_CLOUD_NO_FUSED) at max_nodes 4096 and 8192, on the chain-like shape of `fmt` (revolutions of about 3200 nodes),
    alternating rounds of `steps` pushes"""
    n_streams, max_scans = 512, 56
    if fmt == 0x85:
        n_units, data = 4096, feed(16, 2 * 4096, seed=7)
    else:
        n_units = FORMATS[fmt][2]
        data = feed_format(fmt, 16, 2 * n_units, seed=7)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    cs = stream.cuda_stream
    NS = n_streams * max_scans
    configs = [("push", None), ("window", {}), ("voxel", dict(voxel_size=0.05)),
               ("voxel_separate", dict(voxel_size=0.05, flags=R.CLOUD_NO_FUSED)),
               ("sor_voxel", dict(sor_k=8, sor_alpha=1.0, voxel_size=0.05)),
               ("sor_voxel_separate", dict(sor_k=8, sor_alpha=1.0, voxel_size=0.05, flags=R.CLOUD_NO_FUSED))]
    res = {"format": hex(fmt), "streams": n_streams, "units_per_push": n_units, "max_scans": max_scans, "steps": steps,
           "rounds": rounds, "by_max_nodes": []}
    for max_nodes in (4096, 8192):
        ctx = R.Context(0, max_nodes, NS)
        with torch.cuda.stream(stream):
            halves = [torch.from_numpy(np.ascontiguousarray(np.tile(data[:, h * n_units:(h + 1) * n_units],
                                                                    (n_streams // 16, 1, 1)))).to(dev) for h in (0, 1)]
            d_cnt = torch.full((n_streams,), n_units, dtype=torch.int32, device=dev)
            r = torch.empty((NS, max_nodes), device=dev)
            it = torch.empty((NS, max_nodes), device=dev)
            bc = torch.zeros(NS, dtype=torch.int32, device=dev)
            inc = torch.zeros(NS, device=dev)
            sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
            xyzi = torch.empty((NS, max_nodes, 4), device=dev)
            pc = torch.zeros(NS, dtype=torch.int32, device=dev)
        stream.synchronize()
        row = {"max_nodes": max_nodes, "ms": {k: [] for k, _ in configs}}
        points = {}
        with R.CapsuleStreamSession(ctx, fmt, n_streams, n_units, max_nodes, max_scans) as sess:
            def step_fn(prm):
                def step(t):
                    sess.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                                  bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=cs)
                    if prm is not None:
                        sess.cloud_dev(prm, xyzi.data_ptr(), pc.data_ptr(), stream=cs)
                return step

            fns = {k: step_fn(None if kw is None else R.cloud_params(range_min=0.15, range_max=40.0, **kw))
                   for k, kw in configs}
            for _ in range(rounds):
                for k, _ in configs:
                    row["ms"][k].append(timed(torch, stream, fns[k], steps))
                    if k != "push":
                        points[k] = int(pc.sum().item())
            row["scans_per_push"] = int(sps.sum().item())
            row["scan_nodes_per_push"] = int(bc.sum().item())
        med = {k: float(np.median(v)) for k, v in row["ms"].items()}
        row["ms_median"] = med
        row["cloud_ms_median"] = {k: med[k] - med["push"] for k, _ in configs[1:]}
        # points into the cloud chain (the window's points) and out of it, per push; points/s of push + cloud
        row["points_in_per_push"] = points["window"]
        row["points_out_per_push"] = points
        row["gpoints_per_s"] = {k: points["window"] / (med[k] * 1e-3) / 1e9 for k, _ in configs[1:]}
        row["fused_over_separate"] = {k: med[k] / med[k + "_separate"] - 1.0 for k in ("voxel", "sor_voxel")}
        res["by_max_nodes"].append(row)
        del halves, r, it, xyzi
        ctx.close()
    return res


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=40, help="timed pushes per latency point")
    ap.add_argument("--steps", type=int, default=20, help="timed pushes of the throughput point")
    ap.add_argument("--format", type=lambda v: int(v, 0), default=0x85, choices=[0x81, 0x82, 0x83, 0x84, 0x85, 0x86],
                    help="answer type (default 0x85: the dense session's latency and throughput points)")
    ap.add_argument("--stamped", action="store_true", help="stamped against unstamped pushes of --format")
    ap.add_argument("--rounds", type=int, default=5, help="--stamped, --bytes: alternating rounds of --steps pushes each")
    ap.add_argument("--bytes", action="store_true", help="byte pushes against framed pushes of --format (not 0x81)")
    ap.add_argument("--cloud", action="store_true",
                    help="push_dev alone against push_dev + cloud_dev (0x85 and 0x84 unless --format is given)")
    args = ap.parse_args()
    import torch

    import rplidar_ros2_driver_b200 as R

    if args.cloud:
        fmts = [args.format] if "--format" in " ".join(sys.argv) else [0x85, 0x84]
        if 0x81 in fmts:
            ap.error("--cloud takes a capsule format")
        print(json.dumps({"gpu": gpu_info(), "cloud": [compare_cloud(R, torch, f, args.steps, args.rounds)
                                                       for f in fmts]}))
        return

    if args.bytes:
        if args.format == 0x81:
            ap.error("--bytes takes a capsule format: 0x81 bytes are the standard-node session's input already")
        print(json.dumps({"gpu": gpu_info(), "bytes": [compare_bytes(R, torch, args.format, args.steps, args.rounds, small)
                                                       for small in (False, True)]}))
        return

    if args.stamped:
        print(json.dumps({"gpu": gpu_info(), "stamped": compare_stamped(R, torch, args.format, args.steps, args.rounds)}))
        return

    if args.format == 0x81:
        print(json.dumps({"gpu": gpu_info(), "comparison": compare_normal(R, torch, args.steps),
                          "latency": normal_latency(R, torch, args.pushes)}))
        return
    if args.format != 0x85:
        print(json.dumps({"gpu": gpu_info(), "comparison": compare_stateless(R, torch, args.format, args.steps)}))
        return

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    params = R.scan_params(1, 0, 0, 1)
    res = {"gpu": gpu_info(), "latency": [], "throughput": None}
    n_streams, max_nodes, max_scans = 512, 4096, 16
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    for per in (8, 80, 800):
        caps = feed(16, per * (args.pushes + 4), seed=per)  # 16 distinct streams, tiled over the 512
        rep = n_streams // 16
        counts = np.full(n_streams, per, np.uint32)
        row = {"streams": n_streams, "capsules_per_push": per}
        # host buffers: wall clock around the synchronous call (pinned buffers, as an aggregator would keep them)
        with R.DenseStreamSession(ctx, n_streams, per, max_nodes, max_scans) as sess:
            pin = torch.empty((n_streams, per, 84), dtype=torch.uint8).pin_memory().numpy()
            out = pinned_outputs(torch, n_streams, max_nodes, max_scans)
            ts = []
            for t in range(args.pushes + 4):
                pin[:] = np.tile(caps[:, t * per:(t + 1) * per], (rep, 1, 1))
                t0 = time.perf_counter()
                sess.push(pin, counts, params, out=out)
                ts.append(time.perf_counter() - t0)
            ts = np.array(ts[4:]) * 1e3
            row["push_ms_median"], row["push_ms_p90"] = float(np.median(ts)), float(np.percentile(ts, 90))
        # device buffers: CUDA events around push_dev on a torch stream
        with R.DenseStreamSession(ctx, n_streams, per, max_nodes, max_scans) as sess, torch.cuda.stream(stream):
            d_caps = torch.from_numpy(caps).to(dev)
            d_cnt = torch.full((n_streams,), per, dtype=torch.int32, device=dev)
            NS = n_streams * max_scans
            r = torch.empty((NS, max_nodes), device=dev)
            it = torch.empty((NS, max_nodes), device=dev)
            bc = torch.zeros(NS, dtype=torch.int32, device=dev)
            inc = torch.zeros(NS, device=dev)
            sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.pushes + 4)]
            for t in range(args.pushes + 4):
                piece = d_caps[:, t * per:(t + 1) * per].repeat(rep, 1, 1)
                evs[t][0].record(stream)
                sess.push_dev(piece.data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(), bc.data_ptr(),
                              inc.data_ptr(), sps.data_ptr(), stream=stream.cuda_stream)
                evs[t][1].record(stream)
            stream.synchronize()
            ms = np.array([a.elapsed_time(b) for a, b in evs[4:]])
            row["push_dev_ms_median"], row["push_dev_ms_p90"] = float(np.median(ms)), float(np.percentile(ms, 90))
        res["latency"].append(row)
    ctx.close()
    # throughput on the chain workload's shape
    n_caps, max_scans = 4096, 56
    ctx = R.Context(0, max_nodes, n_streams * max_scans)
    caps = feed(16, n_caps * 2, seed=7)
    with R.DenseStreamSession(ctx, n_streams, n_caps, max_nodes, max_scans) as sess, torch.cuda.stream(stream):
        halves = [torch.from_numpy(np.tile(caps[:, h * n_caps:(h + 1) * n_caps], (n_streams // 16, 1, 1))).to(dev)
                  for h in (0, 1)]
        d_cnt = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
        NS = n_streams * max_scans
        r = torch.empty((NS, max_nodes), device=dev)
        it = torch.empty((NS, max_nodes), device=dev)
        bc = torch.zeros(NS, dtype=torch.int32, device=dev)
        inc = torch.zeros(NS, device=dev)
        sps = torch.zeros(n_streams, dtype=torch.int32, device=dev)

        def push(t):
            sess.push_dev(halves[t % 2].data_ptr(), d_cnt.data_ptr(), params, r.data_ptr(), it.data_ptr(),
                          bc.data_ptr(), inc.data_ptr(), sps.data_ptr(), stream=stream.cuda_stream)

        for t in range(4):
            push(t)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for t in range(args.steps):
            push(t)
        e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        scans = int(sps.cpu().sum())
    res["throughput"] = {"streams": n_streams, "capsules_per_push": n_caps, "ms_per_push": ms,
                         "gnodes_per_s": n_streams * n_caps * 40 / (ms * 1e-3) / 1e9, "scans_per_push": scans}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
