"""The wire decoders over their whole input domain on the device, bit for bit against the SDK's arithmetic.

The families of tests/test_decode_sweep_pieces.py are built on the device with torch (checksums included) as isolated
two-capsule streams through rpl_decode_capsules_batch_dev, with the entering (lastNodeSyncBit, _last_dist_q2) swept
too, and compared with the restatement sdk_streams2 evaluated on the same device tensors: nodes, node counts, capsule
statuses, node offsets and state_out.  Every output starts as a sentinel, so a word the kernel should not write is
caught as well.

  angle pairs A   every prev start field 0..32767 x step_set() (0-4 deg, +-4 counts of the jump thresholds of the
                  sample durations 15, 31, 63 and 125 us, log-spaced to 360 deg), unwrapped and wrapped; all four XOR
                  formats (every other duration's threshold is met exactly, and +1 count, by "thresholds")
  angle pairs B   every cur field 0..32767 x 64 prev fields
  cabin codes     ultra (major, predict1), (predict1, next major) with major 0, (predict2, next major), at even and odd
                  cabins (cabin 31 reads the next capsule's cabin 0)
  sample codes    express (distance word, offset bits) at every position, every dense u16, every ultra-dense qds in
                  both cabin halves
  smoothing       every scale-0 raw distance x incoming last r-9..r+9, 0 and far; chains that never merge, merge
                  mid-capsule and at once
  thresholds      every breakpoint of the jump threshold over sample durations 1..10^6 reachable by a start-angle
                  step: step = threshold (emits) and threshold + 1 count (discards), one launch per sample duration
  checksums       XOR formats: every byte x its 255 other values (rejected), pairs of equal XOR edits (accepted);
                  HQ: every single-bit flip of all 781 bytes (rejected)
  standard nodes  every valid (byte 0, angle word) record through rpl_decode_normal_batch_dev, and every byte 0 and
                  every check-bit-clear byte 1 between records against the oracle's byte machine

Each family prints its case count, wall time and peak device memory (-s shows them)."""
import numpy as np
import pytest
import torch

from test_decode_sweep_pieces import (CB, FULL_Q16, JUMP_CABINS, PER, ST_BAD_FRAME, ST_CHECKSUM, ST_EMIT, ST_OK, XOR_FORMATS,
                                      cabin_pairs, cabin_pairs_size, checksum_pairs, family_a, family_a_size, family_b,
                                      family_b_size, jump_thresholds, pair_states, pairs_from_fields, payload, sample_pairs,
                                      sample_pairs_size, sdk_standard_nodes, sdk_streams2, seal, smoothing_cases,
                                      standard_byte_machine_stream, standard_records, threshold_fields,
                                      threshold_q8)
from test_gpu_domain_sweeps import Meter

gpu = pytest.mark.gpu

CHUNK = {0x82: 1 << 18, 0x84: 1 << 17, 0x85: 1 << 18, 0x86: 1 << 17}  # pairs per launch (peak memory < 2 GiB)
NODE_FILL = 0x5A5A5A5A5A5A5A5A
WORD_FILL = -0x21524111  # 0xDEADBEEF as an int32


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 8192, 64)
    yield c
    c.close()


def run_pairs(ctx, ans, caps, s_in, last_in, sample_us=31):
    """Decode [P, 2, CB] device capsules as P two-capsule streams and compare every output with the restatement.
    Returns the number of pairs that emitted."""
    P = caps.shape[0]
    dev = caps.device
    per = PER[ans]
    caps = caps.contiguous()
    counts = torch.full((P,), 2, dtype=torch.int32, device=dev)
    nodes = torch.full((P, 2 * per), NODE_FILL, dtype=torch.int64, device=dev)
    ncount = torch.full((P,), WORD_FILL, dtype=torch.int32, device=dev)
    status = torch.full((P, 2), WORD_FILL, dtype=torch.int32, device=dev)
    offs = torch.full((P, 2), WORD_FILL, dtype=torch.int32, device=dev)
    state_in = torch.stack([s_in, last_in], 1).to(torch.int32).contiguous()
    state_out = torch.full((P, 2), WORD_FILL, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_capsules_batch_dev(ans, caps.data_ptr(), counts.data_ptr(), P, 2, sample_us, nodes.data_ptr(),
                                  ncount.data_ptr(), state_in=state_in.data_ptr(), capsule_status=status.data_ptr(),
                                  capsule_node_offset=offs.data_ptr(), state_out=state_out.data_ptr())
    ctx.synchronize()
    en, ecount, est, eso = sdk_streams2(ans, caps, s_in, last_in, sample_us)
    emitted = ecount > 0
    want = torch.where(emitted[:, None], en, torch.full_like(en, NODE_FILL))
    bad = (nodes[:, :per] != want).any(1) | (nodes[:, per:] != NODE_FILL).any(1) | (ncount.long() != ecount)
    bad |= (status.long() != est).any(1) | (offs != 0).any(1)
    bad |= (state_out.long() & 0xFFFFFFFF != eso & 0xFFFFFFFF).any(1)
    if bad.any():
        i = int(torch.nonzero(bad)[0])
        pytest.fail(f"{ans:#x}: {int(bad.sum())} of {P} pairs differ; first pair {i}: fields "
                    f"{caps[i, :, 2:4].tolist() if ans != 0x86 else caps[i, :, 8:10].tolist()}, status "
                    f"{status[i].tolist()} vs {est[i].tolist()}, count {int(ncount[i])} vs {int(ecount[i])}, state "
                    f"{state_out[i].tolist()} vs {eso[i].tolist()}, nodes differ at "
                    f"{torch.nonzero(nodes[i, :per] != want[i]).flatten()[:8].tolist()}")
    return int(emitted.sum())


def sweep(ctx, ans, build, size):
    dev = torch.device("cuda")
    for first in range(0, size, CHUNK[ans]):
        n = min(CHUNK[ans], size - first)
        caps = build(first, n)
        s, last = pair_states(ans, first, n, dev)
        run_pairs(ctx, ans, caps, s, last)
    return size


@gpu
@pytest.mark.parametrize("ans", XOR_FORMATS)
def test_angle_pairs(ctx, ans):
    m = Meter()
    n = sweep(ctx, ans, lambda f, k: family_a(ans, f, k, "cuda"), family_a_size())
    n += sweep(ctx, ans, lambda f, k: family_b(ans, f, k, "cuda"), family_b_size())
    m.report(f"angle pairs A + B {ans:#x}", n)


@gpu
def test_ultra_cabin_codes(ctx):
    m = Meter()
    n = sweep(ctx, 0x84, lambda f, k: cabin_pairs(f, k, "cuda"), cabin_pairs_size())
    m.report("cabin codes 0x84", n * 16)


@gpu
@pytest.mark.parametrize("ans", (0x82, 0x85, 0x86))
def test_sample_codes(ctx, ans):
    m = Meter()
    n = sweep(ctx, ans, lambda f, k: sample_pairs(ans, f, k, "cuda"), sample_pairs_size(ans))
    m.report(f"sample codes {ans:#x}", n * PER[ans])


@gpu
def test_smoothing_chain(ctx):
    m = Meter()
    caps, last = smoothing_cases()
    caps, last = caps.cuda(), last.cuda()
    for s in (0, 1):
        run_pairs(ctx, 0x86, caps, torch.full_like(last, s), last)
    m.report("smoothing 0x86", 2 * caps.shape[0])


@gpu
@pytest.mark.parametrize("ans", sorted(JUMP_CABINS))
def test_jump_thresholds(ctx, ans):
    m = Meter()
    n = 0
    for t_q8, sd in sorted(jump_thresholds(ans).items()):
        t = t_q8 // 4
        if t + 1 > 32767:
            continue
        prev, cur = threshold_fields(t, "cuda")
        caps = pairs_from_fields(ans, prev, cur, torch.arange(prev.numel(), device="cuda") + t)
        z = torch.zeros(prev.numel(), dtype=torch.long, device="cuda")
        emitted = run_pairs(ctx, ans, caps, z, z + 4000, sd)
        assert emitted == prev.numel() // 2, (sd, t)  # threshold emits, threshold + 1 count discards
        n += prev.numel()
    m.report(f"thresholds {ans:#x}", n)


@gpu
@pytest.mark.parametrize("ans", XOR_FORMATS)
def test_xor_checksums(ctx, ans):
    m = Meter()
    caps = checksum_pairs(ans, "cuda")
    z = torch.zeros(caps.shape[0], dtype=torch.long, device="cuda")
    run_pairs(ctx, ans, caps, z, z)
    m.report(f"checksums {ans:#x}", caps.shape[0])


@gpu
def test_hq_crc_bit_flips(ctx, oracle):
    m = Meter()
    rng = np.random.default_rng(83)
    base = torch.from_numpy(oracle.seal_capsules(0x83, rng.integers(0, 256, (1, 781), dtype=np.uint8))).cuda()
    n = 781 * 8
    caps = base.repeat(n + 1, 1)
    k = torch.arange(n, device="cuda")
    caps[k, k // 8] ^= (1 << (k % 8)).to(torch.uint8)
    counts = torch.ones(n + 1, dtype=torch.int32, device="cuda")
    nodes = torch.full((n + 1, 96), NODE_FILL, dtype=torch.int64, device="cuda")
    ncount = torch.full((n + 1,), WORD_FILL, dtype=torch.int32, device="cuda")
    status = torch.full((n + 1,), WORD_FILL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.decode_capsules_batch_dev(0x83, caps.data_ptr(), counts.data_ptr(), n + 1, 1, 31, nodes.data_ptr(),
                                  ncount.data_ptr(), capsule_status=status.data_ptr())
    ctx.synchronize()
    want = torch.where(k < 8, ST_BAD_FRAME, ST_CHECKSUM)
    assert (status[:n].long() == want).all() and (ncount[:n] == 0).all() and (nodes[:n] == NODE_FILL).all()
    assert int(status[n]) == ST_OK | ST_EMIT and int(ncount[n]) == 96  # the unflipped capsule
    assert (nodes[n].cpu().numpy().view(np.uint8) == base[0, 9:777].cpu().numpy()).all()
    m.report("checksums 0x83", n + 1)


@gpu
def test_standard_nodes(ctx, oracle):
    m = Meter()
    rec = standard_records("cuda")
    n_streams = 64
    per = rec.shape[0] // n_streams
    stride = per * 5
    wire = rec.reshape(n_streams, stride).contiguous()
    counts = torch.full((n_streams,), stride, dtype=torch.int32, device="cuda")
    nodes = torch.full((n_streams, per), NODE_FILL, dtype=torch.int64, device="cuda")
    ncount = torch.full((n_streams,), WORD_FILL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.decode_normal_batch_dev(wire.data_ptr(), counts.data_ptr(), n_streams, stride, nodes.data_ptr(),
                                ncount.data_ptr())
    ctx.synchronize()
    assert (ncount == per).all()
    want = sdk_standard_nodes(rec).view(n_streams, per)
    assert (nodes == want).all()
    # every byte 0 value and every byte 1 with its check bit clear between valid records, against the byte machine
    b = standard_byte_machine_stream()
    en, _, _ = oracle.decode_normal(b)
    d = torch.from_numpy(b).cuda()
    cnt = torch.tensor([b.size], dtype=torch.int32, device="cuda")
    out = torch.full((b.size // 5,), NODE_FILL, dtype=torch.int64, device="cuda")
    oc = torch.full((1,), WORD_FILL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.decode_normal_batch_dev(d.data_ptr(), cnt.data_ptr(), 1, b.size, out.data_ptr(), oc.data_ptr())
    ctx.synchronize()
    assert int(oc[0]) == len(en)
    assert (out[: len(en)].cpu().numpy() == en.view(np.int64)).all() and (out[len(en):] == NODE_FILL).all()
    m.report("standard nodes 0x81", rec.shape[0] + b.size)


# ---- long streams: the chains across capsules, warps and tiles, against the oracle ------------------------------------
DT = {0x82: 256, 0x84: 256, 0x85: 256, 0x86: 128}  # capsules per tile of decode_capsule_kernel<F>


def capsule_rows(ans, n, seed):
    """[n, CB] payload capsules (unsealed)"""
    return payload(ans, torch.arange((n + 1) // 2) + seed).reshape(-1, CB[ans])[:n].clone()


def chain_streams(ans):
    """The scan-start chain: per sample position p and entering flag, a stream of 2 DT + 40 capsules whose target
    capsules (released at lanes 1, 31, 0 of warp 2, tile positions DT - 2 and 0, and lane 0 of the next tile's second
    warp) have their first raw scan start at sample p, the capsule before each target non-emitting in three ways (none
    for the first), background capsules 0.25 deg apart in between."""
    per, dt = PER[ans], DT[ans]
    n = 2 * dt + 40
    inc = (256 * 256) // per  # the step per sample of a 1 deg (64-count) capsule step
    targets = (0, 30, 63, dt - 3, dt - 1, dt + 31)
    streams, states = [], []
    for p in range(per):
        f = -(-(FULL_Q16 - (p + 1) * inc) // 1024)  # a + (p + 1) inc reaches 360 deg first at sample p
        for s_in in (0, 1):
            v = len(streams)
            caps = capsule_rows(ans, n, 1000 * v + ans)
            fields = 2000 + 16 * torch.arange(n)
            sync = torch.zeros(n, dtype=torch.long)
            kind = v % 4
            for t in targets:
                fields[t], fields[t + 1] = f, f + 64
                if t > 0 and kind == 2:
                    sync[t - 1] = 1
                if t > 0 and kind == 3:
                    fields[t - 1] = (f + 11520) % 23040
            seal(ans, caps, fields, sync)
            if kind == 1:
                for t in targets[1:]:
                    caps[t - 1, 0] ^= 1
            streams.append(caps.numpy())
            states.append((s_in, 0))
    return streams, states


def smoothing_streams():
    """Ultra-dense near-range chains that never merge inside a capsule (equal scale-0 samples, the next capsule within
    8 of them), across capsule, warp and tile boundaries, with checksum errors, scan-start capsules and discarded jumps
    between, entering with last distances 0, near and far."""
    n = 2 * 128 + 40
    streams, states = [], []
    rng = np.random.default_rng(86)
    for v in range(24):
        r = int(rng.integers(100, 1000)) * 4
        step = torch.from_numpy(rng.integers(-1, 2, n)).long() * 4
        qds = (r + torch.cumsum(step, 0) % 8) & 0xFFC  # neighbouring capsules within 8 counts of dist_q2 / 2
        caps = capsule_rows(0x86, n, 5000 + v)
        q = (qds[:, None] | (((torch.arange(n)[:, None] * 3 + torch.arange(64)[None, :]) % 256) << 12)).expand(n, 64)
        cab = caps[:, 10:170].view(n, 32, 5)
        cab[:, :, 0], cab[:, :, 1] = (q[:, 0::2] & 0xFF).to(torch.uint8), ((q[:, 0::2] >> 8) & 0xFF).to(torch.uint8)
        cab[:, :, 2], cab[:, :, 3] = (q[:, 1::2] & 0xFF).to(torch.uint8), ((q[:, 1::2] >> 8) & 0xFF).to(torch.uint8)
        cab[:, :, 4] = ((q[:, 0::2] >> 16) | ((q[:, 1::2] >> 16) << 4)).to(torch.uint8)
        fields = 3000 + 16 * torch.arange(n)
        sync = torch.zeros(n, dtype=torch.long)
        odd = rng.choice(np.arange(2, n - 1), 6, replace=False)
        sync[int(odd[0])] = 1
        fields[int(odd[1])] = (fields[int(odd[1]) + 1] + 11520) % 23040
        seal(0x86, caps, fields, sync)
        caps[int(odd[2]), 0] ^= 1
        streams.append(caps.numpy())
        states.append((v % 2, (0, 2 * r, 2 * r + 8, 1 << 19)[v % 4]))
    return streams, states


def run_streams(ctx, O, ans, streams, states):
    from test_gpu_decode_layout import check_batch, decode, lay_out

    stride = max(len(c) for c in streams)
    L = lay_out(streams, CB[ans], PER[ans], stride, 0, 0, 2, states)
    decode(ctx, ans, "capsules", L)
    check_batch(O, ans, L, [O.decode_capsules(ans, c, 31, st) for c, st in zip(streams, states)])


@gpu
@pytest.mark.parametrize("ans", sorted(JUMP_CABINS))
def test_scan_start_chain(ctx, oracle, ans):
    m = Meter()
    streams, states = chain_streams(ans)
    run_streams(ctx, oracle, ans, streams, states)
    m.report(f"scan-start chain {ans:#x}", len(streams))


@gpu
def test_smoothing_chain_streams(ctx, oracle):
    m = Meter()
    streams, states = smoothing_streams()
    run_streams(ctx, oracle, 0x86, streams, states)
    m.report("smoothing chains 0x86", len(streams))


# ---- the session (STREAM) instantiation ---------------------------------------------------------------------------
SESSION_US = (15, 31, 63, 125)  # per stream, through set_lidars


def session_pairs(ans, sd):
    """The edge pairs a stream session sees: start fields >= 360 deg, zero and negative steps, the stream's jump
    threshold and one count above it, ultra cabin 31, ultra-dense smoothing carries."""
    prev = torch.tensor([23040, 32767, 30000, 5000, 22950, 5000, 26000, 100, 22950, 23100, 22950])
    cur = torch.tensor([23100, 100, 5000, 5000, 23064, 5064, 2000, 32767, 23064, 23040, 23064])  # 22950 -> 23064: a
    # 1.8 deg step across 360 deg (a scan-start node in every format, so that scans close)
    out = [pairs_from_fields(ans, prev, cur, torch.arange(prev.numel()) + 77)]
    if ans in JUMP_CABINS:
        t = threshold_q8(ans, sd) // 4
        if t + 1 <= 32767:
            out.append(pairs_from_fields(ans, *threshold_fields(t), torch.arange(4) + 99))
    if ans == 0x84:
        out.append(cabin_pairs(1, 3))  # odd-parity pairs: cabin 31 reads the next capsule
    if ans == 0x86:
        caps, _ = smoothing_cases()
        out.append(caps[::997][:8])
    return torch.cat(out)


def session_stream(ans, sd):
    """[scan start, prev0, cur0, prev1, cur1, ..., a scan start every 4 pairs]: each pair's prev ends a push and its
    cur opens the next.  Returns the push pieces."""
    pairs = session_pairs(ans, sd)
    start = pairs_from_fields(ans, torch.tensor([0]), torch.tensor([64]), torch.tensor([5]))[0, 0].clone()
    seal(ans, start, torch.tensor(0), torch.tensor(1))
    pieces, cur = [], [start.numpy()]
    for i in range(pairs.shape[0]):
        cur.append(pairs[i, 0].numpy())
        pieces.append(np.stack(cur))
        cur = [pairs[i, 1].numpy()]
        if i % 4 == 3:
            cur.append(start.numpy())
    cur.append(start.numpy())
    pieces.append(np.stack(cur))
    return pieces


@gpu
@pytest.mark.parametrize("ans", XOR_FORMATS)
def test_session_pushes(R, ctx, oracle, ans):
    """Per stream its own sample duration through set_lidars (the session's per-stream jump threshold), every pair
    straddling a push boundary; nodes(apply_ascend=False) of every published scan against the oracle's decode and
    assembly of the whole stream."""
    m = Meter()
    max_nodes, max_scans = 8192, 16
    streams = [session_stream(ans, sd) for sd in SESSION_US]
    n_push = max(len(p) for p in streams)
    stride = max(len(x) for p in streams for x in p)
    got = [[] for _ in SESSION_US]
    with R.CapsuleStreamSession(ctx, ans, len(SESSION_US), stride, max_nodes, max_scans) as sess:
        sess.set_lidars([R.lidar_settings(1, 0, 0, R.Timing(sd, 0, 0, 0)) for sd in SESSION_US])
        params = R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM)
        for k in range(n_push):
            buf = np.zeros((len(SESSION_US), stride, CB[ans]), np.uint8)
            cnt = np.zeros(len(SESSION_US), np.uint32)
            for s, p in enumerate(streams):
                if k < len(p):
                    buf[s, : len(p[k])], cnt[s] = p[k], len(p[k])
            out = sess.push(buf, cnt, params)
            bufs, _ = sess.nodes(apply_ascend=False)
            for s in range(len(SESSION_US)):
                for j in range(min(int(out["scans_per_stream"][s]), max_scans)):
                    got[s].append(np.ascontiguousarray(bufs[s * max_scans + j]).view(np.uint64).copy())
    total = 0
    for s, sd in enumerate(SESSION_US):
        whole = np.concatenate(streams[s])
        nodes, status, offs, _ = oracle.decode_capsules(ans, whole, sd)
        sc, ln, k = oracle.assemble_scans(nodes, oracle.resets_from_capsules(status, offs), max_nodes, 256)
        assert k >= 2 and len(got[s]) == k, (hex(ans), sd, len(got[s]), k)
        for j in range(k):
            assert (got[s][j] == sc[j, : ln[j]].view(np.uint64)).all(), (hex(ans), sd, j)
        if ans in JUMP_CABINS and threshold_q8(ans, sd) // 4 + 1 <= 32767:
            assert (status & oracle.CAPSULE_DISCARD).any()  # the threshold + 1 pair is discarded
        total += len(whole)
    m.report(f"session pushes {ans:#x}", total)
