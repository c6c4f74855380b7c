"""The wire decoders' arithmetic over its whole input domain: the pieces, checked without a GPU.

decode_formats.cu computes reformulations of the SDK's per-capsule arithmetic (a packed-constant varbitscale, a
branchless ultra-dense range decode, running remainders for the scan-start test, a word-folded XOR checksum, the
nine-candidate smoothing chain).  This file holds

  * a plain restatement of the SDK's arithmetic in torch (sdk_pairs, sdk_standard_nodes), written from the SDK lines
    oracle/capsule_oracle.cpp cites, not from the kernel: int64 integer work, the SDK's varbitscale loop,
    k2 = 98361 // dist, the angle offset evaluated per node in float64 in the SDK's order, and the lastNodeSyncBit /
    _last_dist_q2 recurrences as a loop over sample positions, vectorised over capsule pairs.  It runs on CPU and device
    tensors, so tests/test_gpu_decode_sweeps.py checks the kernels against it on the device;
  * the builders of the sweep families, the same torch code on either device;
  * the restatement pinned bit for bit against oracle.decode_capsules and against the SDK's own unpacker on a sample
    of every family (pairs in one byte stream separated by bad-checksum capsules, so that the SDK's previous-capsule
    flag drops while its scan-start bit and last distance carry on);
  * the branches of the kernel's formulations the families reach, and numpy models of those formulations with planted
    faults the families' checkers must reject."""
from __future__ import annotations

import functools
import numpy as np
import pytest
import torch

from reference_outputs import Reference, same
from test_decode_oracle_vs_ref import expected_events

CB = {0x82: 84, 0x83: 781, 0x84: 132, 0x85: 84, 0x86: 170}
PER = {0x82: 32, 0x84: 96, 0x85: 40, 0x86: 64}
START = {0x82: 2, 0x84: 2, 0x85: 2, 0x86: 8}   # byte offset of the start-angle word
JUMP_CABINS = {0x85: 40, 0x86: 32}             # the angular-jump threshold's point count (dense, ultra-dense)
XOR_FORMATS = (0x82, 0x84, 0x85, 0x86)
FULL_Q8 = 360 << 8
FULL_Q16 = 360 << 16
ST_OK, ST_SYNC, ST_EMIT, ST_DISCARD, ST_CHECKSUM, ST_ENC_RESET, ST_BAD_FRAME = 1, 2, 4, 8, 16, 32, 64
SAMPLE_US = (15, 31, 63, 125)


# ---- the SDK's arithmetic, restated ---------------------------------------------------------------------------------
def _u16(c, off):
    return c[:, off].long() | (c[:, off + 1].long() << 8)


def _u32(c, off):
    return _u16(c, off) | (_u16(c, off + 2) << 16)


def _tdiv(a, b):
    """C's integer division (toward zero)."""
    return torch.div(a, b, rounding_mode="trunc")


def _shr(a, k):
    """C's >> on a signed int (arithmetic)."""
    return torch.div(a, 1 << k, rounding_mode="floor")


def _i32(a):
    """The low 32 bits of an int64 as a C int."""
    return ((a + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def _xor_reduce(x):
    """XOR of the last dimension."""
    while x.shape[-1] > 1:
        if x.shape[-1] % 2:
            x = torch.cat([x, torch.zeros_like(x[..., :1])], -1)
        x = x[..., 0::2] ^ x[..., 1::2]
    return x[..., 0]


def threshold_q8(ans, sample_us):
    """maxDiffAngleThreshold_q8 (handler_capsules.cpp:750, :968)."""
    return (360 * 100 * JUMP_CABINS[ans] // (1000000 // int(sample_us))) << 8


def hq_node(angle_q6, dist_q2, sync, quality):
    """The node the SDK publishes, as the u64 of its 8 bytes (angle_z_q14 u16, dist_mm_q2 u32, quality u8, flag u8):
    one wrap of the angle into [0, 360) deg each way, then the (u16) (angle << 8) / 90."""
    a = torch.where(angle_q6 < 0, angle_q6 + (360 << 6), angle_q6)
    a = torch.where(a >= (360 << 6), a - (360 << 6), a)
    key = _tdiv(a << 8, 90) & 0xFFFF
    flag = sync | ((1 - sync) << 1)
    return key | ((dist_q2 & 0xFFFFFFFF) << 16) | ((quality & 0xFF) << 48) | (flag << 56)


def start_q8(ans, c):
    return (_u16(c, START[ans]) & 0x7FFF) << 2


def angle_diff_q8(ans, prev, cur):
    """diffAngle_q8 with the SDK's "+360 deg" when the previous start angle is the larger."""
    p, q = start_q8(ans, prev), start_q8(ans, cur)
    d = q - p
    return torch.where(p > q, d + FULL_Q8, d), p


def varbitscale_decode(scaled):
    """_varbitscale_decode (handler_capsules.cpp:422-458): the first segment base the value reaches, in the SDK's
    order.  Returns (value, level)."""
    value = torch.zeros_like(scaled)
    level = torch.zeros_like(scaled)
    done = torch.zeros_like(scaled, dtype=torch.bool)
    for base, lvl, target in ((3328, 4, 1 << 14), (1792, 3, 1 << 12), (1280, 2, 1 << 11), (512, 1, 1 << 9), (0, 0, 0)):
        remain = scaled - base
        hit = ~done & (remain >= 0)
        value = torch.where(hit, target + remain * (1 << lvl), value)
        level = torch.where(hit, torch.full_like(level, lvl), level)
        done |= hit
    return value, level


def ultra_distances(prev, cur):
    """dist_q2 of the 96 samples of an ultra capsule (handler_capsules.cpp:482-536) [P, 96], int (may be negative)."""
    out = []
    for pos in range(32):
        x3 = _u32(prev, 4 + 4 * pos)
        nx = _u32(cur, 4) if pos == 31 else _u32(prev, 8 + 4 * pos)
        major, lvl1 = varbitscale_decode(x3 & 0xFFF)
        major2, lvl2 = varbitscale_decode(nx & 0xFFF)
        p1 = (x3 >> 12) & 0x3FF
        p1 = torch.where(p1 >= 512, p1 - 1024, p1)
        p2 = (x3 >> 22) & 0x3FF
        p2 = torch.where(p2 >= 512, p2 - 1024, p2)
        borrow = (major == 0) & (major2 != 0)
        base1 = torch.where(borrow, major2, major)
        lvl1 = torch.where(borrow, lvl2, lvl1)
        d0 = major << 2
        d1 = torch.where((p1 == -512) | (p1 == 511), torch.zeros_like(p1), _i32((_i32(p1 * (1 << lvl1)) + base1) * 4))
        d2 = torch.where((p2 == -512) | (p2 == 511), torch.zeros_like(p2), _i32((_i32(p2 * (1 << lvl2)) + major2) * 4))
        out += [d0, d1, d2]
    return torch.stack(out, 1)


def ultra_dense_sample(prev, pos):
    """(raw dist_q2 before smoothing, scale, quality) of sample `pos` (handler_capsules.cpp:984-1017)."""
    cab = 10 + 5 * (pos >> 1)
    hi = prev[:, cab + 4].long()
    qds = _u16(prev, cab + 2 * (pos & 1)) | (((hi >> 4) if pos & 1 else (hi & 0xF)) << 16)
    scale = qds & 3
    dist = torch.where(scale == 0, (qds & 0xFFC) * 2,
                       torch.where(scale == 1, (qds & 0x1FFC) * 3 + (2046 << 2),
                                   torch.where(scale == 2, (qds & 0x3FFC) * 4 + (8187 << 2),
                                               (qds & 0x7FFC) * 5 + (24567 << 2))))
    quality = torch.where(scale == 0, qds >> 12,
                          torch.where(scale == 1, (qds >> 13) << 1,
                                      torch.where(scale == 2, (qds >> 14) << 2, (qds >> 15) << 3))) & 0xFF
    return dist, scale, quality


def sdk_pairs(ans, prev, cur, s_in=None, last_in=None, sample_us=31):
    """The SDK's decode of capsule `prev` when `cur` follows it, for a batch of pairs (uint8 [P, CB] each, both with
    valid checksums and no scan-start bit on `cur`).  s_in / last_in: the lastNodeSyncBit / _last_dist_q2 entering
    (dense, ultra-dense).  Returns (nodes int64 [P, PER] -- the u64 of each node, emitted bool [P], discarded bool [P],
    s_out [P], last_out [P]); nodes of pairs that do not emit are 0 and their state passes through."""
    P, dev = prev.shape[0], prev.device
    z = torch.zeros(P, dtype=torch.long, device=dev)
    s = z.clone() if s_in is None else s_in.long().clone()
    last = z.clone() if last_in is None else last_in.long().clone()
    diff, pq8 = angle_diff_q8(ans, prev, cur)
    a = pq8 << 8
    nodes = []
    if ans == 0x82:  # handler_capsules.cpp:206-266
        inc = diff * 8
        for pos in range(16):
            cab = 4 + 5 * pos
            da = (_u16(prev, cab), _u16(prev, cab + 2))
            ob = prev[:, cab + 4].long()
            offs = ((ob & 0xF) | ((da[0] & 3) << 4), (ob >> 4) | ((da[1] & 3) << 4))
            for c in range(2):
                dist = da[c] & 0xFFFC
                angle = _shr(a - (offs[c] << 13), 10)
                sync = (torch.fmod(a + inc, FULL_Q16) < inc).long()
                a = a + inc
                nodes.append(hq_node(angle, dist, sync, torch.where(dist != 0, 0x2F << 2, 0)))
        emitted = torch.ones(P, dtype=torch.bool, device=dev)
    elif ans == 0x84:  # handler_capsules.cpp:460-580
        inc = _tdiv(diff * 8, 3)
        dist = ultra_distances(prev, cur)
        for i in range(96):
            d = dist[:, i]
            sync = (torch.fmod(a + inc, FULL_Q16) < inc).long()
            off_q16 = torch.full_like(d, int(7.5 * 3.1415926535 * (1 << 16) / 180.0))
            far = d >= 50 * 4
            k2 = torch.where(far, _tdiv(torch.full_like(d, 98361), torch.where(far, d, 1)), 0)
            off_q16 = torch.where(far, int(8 * 3.1415926535 * (1 << 16) / 180) - (k2 << 6) - _tdiv(k2 * k2 * k2, 98304),
                                  off_q16)
            corr = ((off_q16 * 180).double() / 3.14159265).trunc().long()
            angle = _shr(a - corr, 10)
            a = a + inc
            nodes.append(hq_node(angle, d, sync, torch.where(d != 0, 0x2F << 2, 0)))
        emitted = torch.ones(P, dtype=torch.bool, device=dev)
    else:  # dense handler_capsules.cpp:736-791, ultra-dense :951-1047
        n = PER[ans]
        emitted = diff <= threshold_q8(ans, sample_us)
        inc = _tdiv(diff * 256, n)
        s0, last0 = s.clone(), last.clone()
        for pos in range(n):
            if ans == 0x85:
                dist = _u16(prev, 4 + 2 * pos) << 2
                quality = torch.where(dist != 0, 0x2F << 2, 0)
            else:
                dist, scale, quality = ultra_dense_sample(prev, pos)
                near = (scale == 0) & (last != 0) & ((dist - last).abs() <= 8)
                dist = torch.where(near, (dist + last) >> 1, dist)
                last = dist
            angle = _shr(a, 10)
            raw = (torch.fmod(a + inc, FULL_Q16) < inc * 2).long()
            sync = raw & (raw ^ s)
            a = a + inc
            nodes.append(hq_node(angle, dist, sync, quality))
            s = sync
        s = torch.where(emitted, s, s0)
        last = torch.where(emitted, last, last0)
    out = torch.stack(nodes, 1)
    out = torch.where(emitted[:, None], out, torch.zeros_like(out))
    return out, emitted, ~emitted, s, last


def sdk_standard_nodes(rec):
    """The node of each valid 5-byte standard record [P, 5] (handler_normalnode.cpp:115-134), as its u64."""
    rec = rec.long()
    angle_chk = rec[:, 1] | (rec[:, 2] << 8)
    key = ((angle_chk >> 1) << 8) // 90 & 0xFFFF
    dist = rec[:, 3] | (rec[:, 4] << 8)
    return key | (dist << 16) | (((rec[:, 0] >> 2) << 2) << 48) | ((rec[:, 0] & 1) << 56)


def capsule_frame_status(ans, caps):
    """(checksum ok, status of the capsule on its own) for [P, CB]: the sync nibbles, then the XOR of bytes 2.. (CRC32
    for HQ is not restated here)."""
    b0, b1 = caps[:, 0].long(), caps[:, 1].long()
    framed = ((b0 >> 4) == 0xA) & ((b1 >> 4) == 0x5)
    x = _xor_reduce(caps[:, 2:CB[ans]].long())
    ok = framed & (x == ((b0 & 0xF) | ((b1 & 0xF) << 4)))
    st = torch.where(framed, torch.where(ok, ST_OK, ST_CHECKSUM), ST_BAD_FRAME)
    return ok, st


def sdk_streams2(ans, caps, s_in, last_in, sample_us=31):
    """Two-capsule streams [P, 2, CB] as the SDK decodes them: (nodes [P, PER], node count [P], status [P, 2],
    state_out [P, 2]) in the layout of rpl_decode_capsules_batch_dev.  The first capsule has no predecessor."""
    prev, cur = caps[:, 0], caps[:, 1]
    ok0, st0 = capsule_frame_status(ans, prev)
    ok1, st1 = capsule_frame_status(ans, cur)
    sy0 = ok0 & ((_u16(prev, START[ans]) >> 15) == 1)
    sy1 = ok1 & ((_u16(cur, START[ans]) >> 15) == 1)
    st0 = st0 | torch.where(sy0, ST_SYNC, 0)
    st1 = st1 | torch.where(sy1, ST_SYNC, 0) | torch.where(sy1 & ok0, ST_ENC_RESET, 0)
    go = ok0 & ok1 & ~sy1
    nodes, emitted, discarded, s, last = sdk_pairs(ans, prev, cur, s_in, last_in, sample_us)
    emitted, discarded = emitted & go, discarded & go
    st1 = st1 | torch.where(emitted, ST_EMIT, 0) | torch.where(discarded, ST_DISCARD, 0)
    nodes = torch.where(emitted[:, None], nodes, torch.zeros_like(nodes))
    s_in = torch.zeros_like(s) if s_in is None else s_in.long()
    last_in = torch.zeros_like(last) if last_in is None else last_in.long()
    s = torch.where(emitted, s, s_in) if ans in (0x85, 0x86) else torch.zeros_like(s)
    last = torch.where(emitted, last, last_in) if ans == 0x86 else torch.zeros_like(last)
    count = torch.where(emitted, PER[ans], 0)
    return nodes, count, torch.stack([st0, st1], 1), torch.stack([s, last], 1)


# ---- the sweep families ---------------------------------------------------------------------------------------------
def _mix(x):
    """A fixed 32-bit integer hash (payload bytes that differ from case to case)."""
    x = (x * 0x9E3779B1) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x85EBCA77) & 0xFFFFFFFF
    return x ^ (x >> 13)


def seal(ans, caps, start=None, sync=None):
    """Start-angle field (15 bits) and scan-start bit, then the sync nibbles and the XOR checksum, in place on
    uint8 [..., CB]."""
    off = START[ans]
    if start is not None:
        w = (start.long() & 0x7FFF) | ((sync.long() if sync is not None else 0) << 15)
        caps[..., off] = (w & 0xFF).to(torch.uint8)
        caps[..., off + 1] = (w >> 8).to(torch.uint8)
    chk = _xor_reduce(caps[..., 2:].long())
    caps[..., 0] = (0xA0 | (chk & 0xF)).to(torch.uint8)
    caps[..., 1] = (0x50 | (chk >> 4)).to(torch.uint8)
    return caps


def payload(ans, pair_ids):
    """Payload bytes of both capsules of each pair [P, 2, CB].  Express: the 6-bit angle offsets of the pair's 32
    samples cycle all 64 values across pairs; ultra: the majors of its 32 cabins step through all 4096 codes every 128
    pairs, so every k2 table entry is met; dense / ultra-dense: hashed distance words."""
    P, dev = pair_ids.shape[0], pair_ids.device
    cb = CB[ans]
    idx = pair_ids.long()[:, None, None] * (2 * cb) + torch.arange(2, device=dev)[None, :, None] * cb + \
        torch.arange(cb, device=dev)[None, None, :]
    caps = (_mix(idx) & 0xFF).to(torch.uint8)
    if ans == 0x82:
        j = torch.arange(32, device=dev)
        off = (pair_ids.long()[:, None] + j[None, :]) % 64  # [P, 32]
        for k in range(2):
            cab = caps[:, k, 4:84].view(P, 16, 5)
            cab[:, :, 0] = (cab[:, :, 0] & 0xFC) | (off[:, 0::2] >> 4).to(torch.uint8)
            cab[:, :, 2] = (cab[:, :, 2] & 0xFC) | (off[:, 1::2] >> 4).to(torch.uint8)
            cab[:, :, 4] = ((off[:, 0::2] & 0xF) | ((off[:, 1::2] & 0xF) << 4)).to(torch.uint8)
    elif ans == 0x84:
        code = ((pair_ids.long()[:, None] * 32 + torch.arange(32, device=dev)[None, :]) * 7) % 4096  # [P, 32]
        for k in range(2):
            w = caps[:, k, 4:132].view(P, 32, 4)
            w[:, :, 0] = (code & 0xFF).to(torch.uint8)
            w[:, :, 1] = ((w[:, :, 1].long() & 0xF0) | (code >> 8)).to(torch.uint8)
    return caps


def pairs_from_fields(ans, prev_field, cur_field, pair_ids=None):
    """Sealed pairs [P, 2, CB] with the given start fields (0..32767) and the family payload."""
    if pair_ids is None:
        pair_ids = torch.arange(prev_field.shape[0], device=prev_field.device)
    caps = payload(ans, pair_ids)
    seal(ans, caps[:, 0], prev_field)
    seal(ans, caps[:, 1], cur_field)
    return caps


def jump_thresholds(ans, lo=1, hi=1000000):
    """{threshold_q8: the smallest sample duration giving it} over sample durations lo..hi: every breakpoint."""
    sd = np.arange(lo, hi + 1, dtype=np.int64)
    thr = (360 * 100 * JUMP_CABINS[ans] // (1000000 // sd)) << 8
    first = np.flatnonzero(np.diff(thr, prepend=-1) != 0)
    return {int(thr[i]): int(sd[i]) for i in first}


def step_set():
    """The family-A steps in q6 units (start-field counts): every step of 0..4 deg, every step within 4 counts of the
    jump thresholds of the common sample durations (the threshold family takes every other duration's threshold and
    threshold + 1 count), 64 log-spaced steps up to 360 deg, 359.98 and 360 deg."""
    steps = set(range(257))
    for ans in (0x85, 0x86):
        for sd in SAMPLE_US:
            t = threshold_q8(ans, sd)
            steps.update(range(t // 4 - 4, t // 4 + 5))
    steps.update(np.unique(np.round(np.geomspace(1, 360 * 64, 64))).astype(int).tolist())
    steps.update((360 * 64 - 1, 360 * 64))
    return torch.tensor(sorted(s for s in steps if 0 <= s <= 32767), dtype=torch.long)


def threshold_fields(t, device="cpu"):
    """(prev, cur) start fields whose step is t and t + 1 counts: unwrapped from 0, and wrapped from 23039 where the
    step is below 360 deg."""
    prev = [0, 0] + ([23039, 23039] if t + 1 < 23039 else [])
    cur = [t, t + 1] + ([t - 1, t] if t + 1 < 23039 else [])
    return torch.tensor(prev, device=device), torch.tensor(cur, device=device)


def family_a(ans, first, count, device="cpu"):
    """Angle pairs A, cases first..first+count: every prev field 0..32767 x every step of step_set(), unwrapped
    (cur = prev + step) and wrapped (cur = prev + step - 23040); cur fields outside 0..32767 wrap mod 2^15."""
    steps = step_set().to(device)
    k = torch.arange(first, first + count, device=device)
    prev = k % 32768
    j = k // 32768
    step = steps[(j // 2) % steps.numel()]
    cur = torch.where(j % 2 == 0, prev + step, prev + step - 360 * 64) & 0x7FFF
    return pairs_from_fields(ans, prev, cur, k)


def family_a_size():
    return 32768 * 2 * int(step_set().numel())


B_PREV = (0, 1, 63, 64, 11519, 11520, 23039, 23040, 23041, 32767)


def family_b_prev():
    rng = np.random.default_rng(5)
    return torch.tensor(list(B_PREV) + rng.integers(0, 32768, 54).tolist(), dtype=torch.long)


def family_b(ans, first, count, device="cpu"):
    """Angle pairs B: every cur field 0..32767 x 64 prev values (the edges of the field and of 180 / 360 deg)."""
    pv = family_b_prev().to(device)
    k = torch.arange(first, first + count, device=device)
    cur = k % 32768
    prev = pv[k // 32768]
    return pairs_from_fields(ans, prev, cur, k + (1 << 30))


def family_b_size():
    return 32768 * int(family_b_prev().numel())


def family_cabins(first, count, device="cpu"):
    """Ultra cabin codes.  Case k = (kind, code, parity): kind 0 every (major, predict1) with a nonzero next major,
    kind 1 every (predict1, next major) with major 0 (the borrowed base), kind 2 every (predict2, next major).  Each
    pair holds 16 cases, at the even cabins (parity 0) or the odd ones (parity 1: cabin 31 reads the next capsule's
    cabin 0); the cabin after a case supplies its next major.  So each code sits at two cabins, 2 (code % 16) + parity,
    and every cabin 0..31 holds every kind; only cabin 31 (the next major from the next capsule) differs in arithmetic."""
    k = torch.arange(first, first + count, device=device)
    pair = k // 16
    slot = k % 16
    kind = pair // (2 * (1 << 22) // 16)
    within = pair % (2 * (1 << 22) // 16)
    parity = within % 2
    code = (within // 2) * 16 + slot  # 0 .. 2^22 - 1: 12-bit major (or next major) x 10-bit predict
    hi, lo = code >> 10, code & 0x3FF
    h = _mix(k + (3 << 30))
    x3 = torch.where(kind == 0, hi | (lo << 12) | ((h & 0x3FF) << 22),
                     torch.where(kind == 1, (lo << 12) | ((h & 0x3FF) << 22), (h & 0xFFF) | (((h >> 12) & 0x3FF) << 12) | (lo << 22)))
    nxt = torch.where(kind == 0, (h >> 20) | 1, hi) | (((h >> 8) & 0xFFFFF) << 12)
    return pair, parity, x3, nxt


def cabin_pairs(first_pair, n_pairs, device="cpu"):
    pair, parity, x3, nxt = family_cabins(first_pair * 16, n_pairs * 16, device)
    P = n_pairs
    words = torch.zeros(P, 2, 33, dtype=torch.long, device=device)  # prev cabins 0..31, cur cabin 0 (as index 32)
    par = parity.view(P, 16)[:, 0]
    subj = (torch.arange(16, device=device)[None, :] * 2 + par[:, None])  # [P, 16]
    words[:, 0].scatter_(1, subj, x3.view(P, 16))
    words[:, 0].scatter_(1, subj + 1, nxt.view(P, 16))
    caps = payload(0x84, torch.arange(first_pair, first_pair + P, device=device) + (1 << 29))
    w = words[:, 0]
    b = torch.stack([(w >> (8 * i)) & 0xFF for i in range(4)], -1).to(torch.uint8)  # [P, 33, 4]
    caps[:, 0, 4:132] = b[:, :32].reshape(P, 128)
    caps[:, 1, 4:8] = b[:, 32]
    fields = (torch.arange(first_pair, first_pair + P, device=device) * 97) % 23040
    seal(0x84, caps[:, 0], fields)
    seal(0x84, caps[:, 1], (fields + 170) % 23040)
    return caps


def cabin_pairs_size():
    return 3 * 2 * (1 << 22) // 16


def sample_pairs(ans, first, count, device="cpu"):
    """Sample codes.  Express: every (16-bit distance word, 4 offset bits) at every sample position (pair p, sample j
    carries code (p + j) mod 2^20); dense: every u16 distance at every position; ultra-dense: every 20-bit qds in both
    halves of a cabin (half 0 code p * 32 + cabin, half 1 that code XOR 0xA5A5A)."""
    p = torch.arange(first, first + count, device=device)
    caps = payload(ans, p + (1 << 28))
    P = count
    if ans == 0x82:
        j = torch.arange(32, device=device)
        code = (p[:, None] + j[None, :]) % (1 << 20)
        word, nib = code & 0xFFFF, code >> 16
        cab = caps[:, 0, 4:84].view(P, 16, 5)
        cab[:, :, 0], cab[:, :, 1] = (word[:, 0::2] & 0xFF).to(torch.uint8), (word[:, 0::2] >> 8).to(torch.uint8)
        cab[:, :, 2], cab[:, :, 3] = (word[:, 1::2] & 0xFF).to(torch.uint8), (word[:, 1::2] >> 8).to(torch.uint8)
        cab[:, :, 4] = (nib[:, 0::2] | (nib[:, 1::2] << 4)).to(torch.uint8)
    elif ans == 0x85:
        j = torch.arange(40, device=device)
        code = (p[:, None] + j[None, :]) % 65536
        caps[:, 0, 4:84] = torch.stack([code & 0xFF, code >> 8], -1).reshape(P, 80).to(torch.uint8)
    else:
        cab_i = torch.arange(32, device=device)
        q0 = (p[:, None] * 32 + cab_i[None, :]) % (1 << 20)
        q1 = q0 ^ 0xA5A5A
        cab = caps[:, 0, 10:170].view(P, 32, 5)
        cab[:, :, 0], cab[:, :, 1] = (q0 & 0xFF).to(torch.uint8), ((q0 >> 8) & 0xFF).to(torch.uint8)
        cab[:, :, 2], cab[:, :, 3] = (q1 & 0xFF).to(torch.uint8), ((q1 >> 8) & 0xFF).to(torch.uint8)
        cab[:, :, 4] = ((q0 >> 16) | ((q1 >> 16) << 4)).to(torch.uint8)
    fields = (p * 37) % 23040
    seal(ans, caps[:, 0], fields)
    seal(ans, caps[:, 1], (fields + 40) % 23040)
    return caps


def sample_pairs_size(ans):
    return {0x82: 1 << 20, 0x85: 65536, 0x86: 1 << 15}[ans]


def pair_states(ans, first, count, device="cpu"):
    """The (lastNodeSyncBit, _last_dist_q2) entering each pair: both sync bits, and for ultra-dense distances near and
    far from the samples (0, a few counts either side of common codes, far)."""
    k = torch.arange(first, first + count, device=device)
    s = (_mix(k + (5 << 30)) & 1).long()
    lasts = torch.tensor([0, 1, 800, 3000, 4092, 8184, 16380, 0xFFFFF], device=device)
    last = lasts[(_mix(k + (6 << 30)) >> 3) % lasts.numel()] if ans == 0x86 else torch.zeros_like(s)
    return s, last


def checksum_pairs(ans, device="cpu"):
    """XOR formats: a valid capsule with one byte changed to each of its 255 other values (rejected), and pairs of bytes
    changed by the same XOR delta (accepted).  Returns caps [P, 2, CB]: a valid first capsule and the edited one."""
    cb = CB[ans]
    base = pairs_from_fields(ans, torch.tensor([1000], device=device), torch.tensor([1100], device=device))[0]
    pos = torch.arange(cb, device=device).repeat_interleave(255)
    delta = torch.arange(1, 256, device=device).repeat(cb)
    one = base[None].repeat(pos.numel(), 1, 1)
    one[torch.arange(pos.numel(), device=device), 1, pos] ^= delta.to(torch.uint8)
    i = torch.arange(2, cb, device=device)
    j = torch.roll(i, 1)
    d = (torch.arange(i.numel(), device=device) * 37) % 255 + 1
    two = base[None].repeat(i.numel() * 2, 1, 1)
    r = torch.arange(i.numel(), device=device)
    two[r, 1, i] ^= d.to(torch.uint8)
    two[r, 1, j] ^= d.to(torch.uint8)
    k = (i + 5 - 2) % (cb - 2) + 2  # a second pattern: pairs further apart, and deltas 0x80 / 0x01
    two[r + i.numel(), 1, i] ^= torch.where(r % 2 == 0, 0x80, 0x01).to(torch.uint8)
    two[r + i.numel(), 1, k] ^= torch.where(r % 2 == 0, 0x80, 0x01).to(torch.uint8)
    return torch.cat([one, two])


def standard_records(device="cpu"):
    """Every valid (byte 0, angle word) record: byte 0 with its sync bit and inverse (128 values) x every angle word with
    its check bit set (32768), hashed distances.  uint8 [2^22, 5]."""
    k = torch.arange(1 << 22, device=device)
    b0 = k >> 15
    b0 = ((b0 >> 1) << 2) | (b0 & 1) | ((1 - (b0 & 1)) << 1)
    w = ((k & 0x7FFF) << 1) | 1
    h = _mix(k + (7 << 30))
    return torch.stack([b0, w & 0xFF, w >> 8, h & 0xFF, (h >> 8) & 0xFF], 1).to(torch.uint8)


def standard_byte_machine_stream(seed=3, n_records=6000):
    """Valid records with every byte-0 value (invalid ones are dropped) and every byte 1 with its check bit clear (the
    record restarts) in between."""
    rng = np.random.default_rng(seed)
    rec = standard_records()[torch.from_numpy(rng.integers(0, 1 << 22, n_records))].numpy()
    out = []
    bad1 = [b for b in range(256) if not b & 1]
    for i in range(n_records):
        out.append(rec[i])
        if i < 256:
            out.append(np.array([i], np.uint8))
        elif i - 256 < len(bad1):
            out.append(np.array([rec[i, 0], bad1[i - 256]], np.uint8))
    return np.concatenate(out)


# ---- sampled streams for the oracle and the SDK -----------------------------------------------------------------------
def bad_capsule(ans, like):
    c = like.clone()
    c[0] ^= 0x01  # the checksum nibble: a checksum error (the SDK drops its previous-capsule flag)
    return c


def prefix(ans):
    """A pair whose nodes hold no scan start (so the SDK's function-static dense sync bit leaves it as 0), then a bad
    capsule: every sampled stream starts from the same SDK state."""
    c = pairs_from_fields(ans, torch.tensor([640]), torch.tensor([1280]), torch.tensor([12345]))[0]
    return [c[0], c[1], bad_capsule(ans, c[1])]


def joined(ans, pairs):
    """[prefix, prev0, cur0, bad, prev1, cur1, bad, ...] as one capsule array."""
    out = prefix(ans)
    for p in range(pairs.shape[0]):
        out += [pairs[p, 0], pairs[p, 1], bad_capsule(ans, pairs[p, 1])]
    return torch.stack(out).numpy()


def restated_stream(ans, pairs, sample_us):
    """What the SDK emits for joined(ans, pairs): the prefix pair, then every pair with the state left by the pairs
    before it.  Returns (nodes [M] u64, status [n], offsets [n])."""
    pre = torch.stack(prefix(ans)[:2])[None]
    allp = torch.cat([pre, pairs])
    s, last = torch.zeros(1, dtype=torch.long), torch.zeros(1, dtype=torch.long)
    nodes, status, offs, n_out = [], [], [], 0
    for p in range(allp.shape[0]):
        nd, cnt, st, so = sdk_streams2(ans, allp[p:p + 1], s, last, sample_us)
        status += [int(st[0, 0]), int(st[0, 1]), ST_CHECKSUM]
        offs += [n_out, n_out, n_out + int(cnt[0])]
        n_out += int(cnt[0])
        nodes.append(nd[0, :int(cnt[0])])
        s, last = so[:, 0], so[:, 1]
    return torch.cat(nodes).numpy().astype(np.uint64), np.array(status, np.uint32), np.array(offs, np.uint32)


def samples(ans):
    """A sample of every family that serves `ans`, as pairs [P, 2, CB] with the sample duration to decode them at."""
    rng = np.random.default_rng(ans)
    out = []
    a = family_a_size()
    # the edges of family A: start fields >= 360 deg, zero and negative steps, thresholds +-1 step
    idx = torch.from_numpy(np.concatenate([rng.integers(0, a, 100), np.arange(23040, 23040 + 24),
                                           np.arange(32768 * 2 - 24, 32768 * 2 + 24)]))
    caps_a = torch.cat([family_a(ans, int(i), 1) for i in idx])
    out.append(("A", caps_a, 31))
    caps_b = torch.cat([family_b(ans, int(i), 1) for i in rng.integers(0, family_b_size(), 60)])
    out.append(("B", caps_b, 31))
    if ans == 0x84:
        out.append(("cabins", torch.cat([cabin_pairs(int(i), 1) for i in rng.integers(0, cabin_pairs_size(), 40)]), 31))
    else:
        n = sample_pairs_size(ans)
        out.append(("samples", torch.cat([sample_pairs(ans, int(i), 1) for i in rng.integers(0, n, 40)]), 31))
    if ans in JUMP_CABINS:
        th = []
        for sd in SAMPLE_US + (1, 7, 355, 1000):
            t = threshold_q8(ans, sd) // 4
            if t + 1 <= 32767:
                th.append((sd, pairs_from_fields(ans, *threshold_fields(t))))
        for sd, c in th:
            out.append((f"threshold sd={sd}", c, sd))
    return out


@pytest.fixture(scope="module")
def ref(oracle):
    return Reference(oracle)


@pytest.mark.parametrize("ans", XOR_FORMATS)
def test_restatement_matches_oracle_and_sdk(ref, ans):
    """Every family's sample, joined into one stream, through the restatement, oracle.decode_capsules and the SDK's
    unpacker: the same nodes, statuses and events."""
    for name, pairs, sd in samples(ans):
        caps = joined(ans, pairs)
        en, es, eo = restated_stream(ans, pairs, sd)
        on, os_, oo, _ = ref.decode_capsules(ans, caps, sd, (0, 0))
        where = (hex(ans), name)
        assert len(on) == len(en), where
        assert (on.view(np.uint64) == en).all(), where
        assert (os_ == es).all() and (oo == eo).all(), where
        rn, rev = ref.ref_unpack(ans, caps.reshape(-1), sd, 0)
        assert len(rn) == len(en) and same(en.view(ref.NODE_DTYPE), rn), where
        exp = expected_events(ref, es, eo)
        assert len(exp) == len(rev) and same(exp, rev), where


def test_pairs_match_oracle_with_entering_state(oracle):
    """Isolated two-capsule streams with every entering state: the restatement's state out is the oracle's."""
    for ans in XOR_FORMATS:
        caps = family_a(ans, 23040 * 3 + 11, 64)
        s, last = pair_states(ans, 0, 64)
        nodes, cnt, st, so = sdk_streams2(ans, caps, s, last)
        for p in range(64):
            on, os_, oo, ost = oracle.decode_capsules(ans, caps[p].numpy(), 31, (int(s[p]), int(last[p])))
            assert len(on) == int(cnt[p]) and (on.view(np.int64) == nodes[p, :len(on)].numpy()).all(), (hex(ans), p)
            assert (os_ == st[p].numpy()).all() and (oo == [0, 0]).all()
            want = {0x85: (ost[0], 0), 0x86: ost}.get(ans, (0, 0))
            assert tuple(int(x) for x in so[p]) == tuple(want), (hex(ans), p)


def test_standard_records_match_oracle(oracle):
    rec = standard_records()
    rng = np.random.default_rng(2)
    pick = torch.from_numpy(rng.integers(0, rec.shape[0], 20000))
    want = sdk_standard_nodes(rec[pick]).numpy()
    nodes, _, pos = oracle.decode_normal(rec[pick].numpy().reshape(-1))
    assert pos == 0 and (nodes.view(np.int64) == want).all()
    nodes, _, _ = oracle.decode_normal(standard_byte_machine_stream())
    assert 5000 < len(nodes) < 6000  # some inserted bytes start records, and the bytes after them are lost


def test_checksum_cases_are_what_they_claim():
    for ans in XOR_FORMATS:
        caps = checksum_pairs(ans)
        ok, st = capsule_frame_status(ans, caps[:, 1])
        n1 = CB[ans] * 255
        assert not ok[:n1].any() and ok[n1:].all()
        assert ((st[:n1] == ST_BAD_FRAME) | (st[:n1] == ST_CHECKSUM)).all()


# ---- branch reach -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def angle_cases():
    """(prev_q8, diff_q8) of every family-A and family-B pair (the start fields do not depend on the format)."""
    steps = step_set()
    prev = torch.arange(32768).repeat(2 * steps.numel())
    j = torch.arange(2 * steps.numel()).repeat_interleave(32768)
    step = steps[j // 2]
    cur = torch.where(j % 2 == 0, prev + step, prev + step - 23040) & 0x7FFF
    pb = family_b_prev().repeat_interleave(32768)
    cb = torch.arange(32768).repeat(family_b_prev().numel())
    p, c = torch.cat([prev, pb]) << 2, torch.cat([cur, cb]) << 2
    d = torch.where(p > c, c - p + FULL_Q8, c - p)
    return p, d


def raw_sync_mask_model(prev_q8, inc, n, exit_le=False, strict_sub=False):
    """raw_sync_mask<N> as the kernel computes it (numpy int64 standing in for int32): one modulo, the early exit, then
    the running remainder.  Returns (masks as a list of bool arrays, early exit taken)."""
    rem = np.fmod((prev_q8 << 8) + inc, FULL_Q16)
    lim = inc << 1
    last = rem + (n - 1) * inc
    ex = (rem >= lim) & ((last <= FULL_Q16) if exit_le else (last < FULL_Q16))
    bits = []
    for pos in range(n):
        bits.append(~ex & (rem < lim))
        rem = rem + inc
        rem = np.where((rem > FULL_Q16) if strict_sub else (rem >= FULL_Q16), rem - FULL_Q16, rem)
    return bits, ex


def raw_sync_sdk(prev_q8, inc, n):
    a = prev_q8 << 8
    return [np.fmod(a + pos * inc + inc, FULL_Q16) < (inc << 1) for pos in range(n)]


def express_sync_model(prev_q8, diff, strict_sub=False):
    """cabin_express's scan-start flags of all 32 samples: per cabin one modulo, the second by the running remainder
    when the step is in [0, 360 deg), else another modulo."""
    inc = diff << 3
    out = []
    for cabin in range(16):
        a0 = (prev_q8 << 8) + 2 * cabin * inc
        a1 = a0 + inc
        rem = np.fmod(a1, FULL_Q16)
        out.append(rem < inc)
        step_ok = (inc >= 0) & (inc < FULL_Q16)
        r2 = rem + inc
        r2 = np.where((r2 > FULL_Q16) if strict_sub else (r2 >= FULL_Q16), r2 - FULL_Q16, r2)
        r2 = np.where(step_ok, r2, np.fmod(a1 + inc, FULL_Q16))
        out.append(r2 < inc)
    return out


def express_sync_sdk(prev_q8, diff):
    inc = diff << 3
    a = prev_q8 << 8
    return [np.fmod(a + pos * inc + inc, FULL_Q16) < inc for pos in range(32)]


def c_div(a, n):
    """C's truncating integer division on numpy int64."""
    return np.where(a < 0, -((-a) // n), a // n)


def test_branch_reach():
    seen = {sc: set() for sc in range(4)}
    p, d = angle_cases()
    p, d = p.numpy(), d.numpy()
    assert (d < 0).any() and (d == 0).any()                                        # negative diff, zero step
    assert ((p >= FULL_Q8) & (d < 0)).any()                                        # prev >= 360 deg + cur
    # raw_sync_mask: early exit taken and not taken, the running remainder's subtraction, for both chained formats
    for n in (40, 64):
        inc = c_div(d << 8, n)
        rem = np.fmod((p << 8) + inc, FULL_Q16)
        ex = (rem >= (inc << 1)) & (rem + (n - 1) * inc < FULL_Q16)  # raw_sync_mask's early exit
        assert ex.any() and (~ex).any()
        assert ((~ex) & (rem + inc >= FULL_Q16)).any()
    # express / ultra: step_ok false only for negative steps, which the families reach
    assert ((d << 3) < 0).any()
    # pack_node: an interpolated angle >= 720 deg (the last ultra-dense sample), and both wraps (express sample 0 below
    # zero when its offset exceeds the start angle; start angles >= 360 deg)
    top = ((p << 8) + 63 * c_div(d << 8, 64)) >> 10
    assert (top >= 2 * (360 << 6)).any()
    assert ((p >> 2) >= (360 << 6)).any()
    caps = family_a(0x82, 0, 64)
    off0 = (caps[:, 0, 8].long() & 0xF) | ((caps[:, 0, 4].long() & 3) << 4)
    assert ((torch.arange(64) * 1024 - (off0 << 13)) < 0).any()
    # ultra: every k2 entry a distance can reach, a negative predicted distance, the short-range default.  Every ultra
    # distance is a multiple of 4 (dist_q2 = value << 2), so k2 = 98361 // (4 n), n >= 50: 265 of the table's 493
    # entries (the others are unreachable from the wire)
    caps = family_a(0x84, 0, 256)
    dist = ultra_distances(caps[:, 0], caps[:, 1]).reshape(-1).numpy()
    k2 = np.where(dist >= 200, 98361 // np.maximum(dist, 1), 492)
    reachable = {98361 // (4 * n) for n in range(50, 98361 // 4 + 2)} | {492}
    assert set(np.unique(k2).tolist()) == reachable, len(reachable)
    assert (dist < 0).any()
    # ultra-dense: every scale on both sides of |raw - last| = 8 (the smoothing and the sample-code families)
    for caps, last in (smoothing_cases(), (sample_pairs(0x86, 0, 2048), torch.zeros(2048, dtype=torch.long))):
        last = last.clone()
        for pos in range(64):
            raw, scale, _ = ultra_dense_sample(caps[:, 0], pos)
            near = (raw - last).abs() <= 8
            for sc in range(4):
                seen[sc] |= {bool(x) for x in torch.unique(near[(scale == sc) & (last != 0)]).tolist()}
            last = torch.where((scale == 0) & (last != 0) & near, (raw + last) >> 1, raw)
    assert all(seen[sc] == {True, False} for sc in range(4)), seen
    # ud_pm in {0, mid, 64}: first scale nonzero -> 0; near chains merge late or never
    pm = ud_merge_positions(smoothing_cases())
    assert (pm == 0).any() and ((pm > 0) & (pm < 64)).any() and (pm == 64).any()


# ---- the smoothing chain --------------------------------------------------------------------------------------------
def smoothing_cases():
    """Ultra-dense capsules for the smoothing chain: every scale-0 raw value r (a multiple of 8) with incoming last
    values r-9..r+9, 0 and far, through one capsule of near samples that never merge (64), of a far sample at a middle
    position, and of a scale-nonzero first sample.  Returns (caps [P, 2, CB], last_in [P])."""
    r = torch.arange(0, 4096, 4) * 2  # every scale-0 raw dist_q2 (qds & 0xFFC) * 2
    lasts = torch.cat([torch.arange(-9, 10), torch.tensor([10 ** 6])])
    R = r.repeat_interleave(lasts.numel() + 1)
    L = torch.cat([r[:, None] + lasts[None, :], torch.zeros(r.numel(), 1, dtype=torch.long)], 1).reshape(-1).clamp(min=0)
    P = R.numel()
    kind = torch.arange(P) % 4
    caps = payload(0x86, torch.arange(P) + (1 << 27))
    pos = torch.arange(64)
    # kind 0: 64 equal scale-0 samples (the candidates settle on two values and never merge); 1: a scale-3 sample at
    # position 31 (they merge there); 2: a scale-1 first sample (merged at once); 3: 64 equal samples of scale 1..3
    v = (R[:, None] // 2).expand(P, 64) & 0xFFC
    v = torch.where((kind[:, None] == 1) & (pos[None, :] == 31), v | 3, v)
    v = torch.where((kind[:, None] == 2) & (pos[None, :] == 0), v | 1, v)
    v = torch.where(kind[:, None] == 3, v | (torch.arange(P)[:, None] // 4 % 3 + 1), v)
    q = v | (((torch.arange(P)[:, None] + pos[None, :] * (kind[:, None] != 3)) % 256) << 12)
    cab = caps[:, 0, 10:170].view(P, 32, 5)
    cab[:, :, 0], cab[:, :, 1] = (q[:, 0::2] & 0xFF).to(torch.uint8), ((q[:, 0::2] >> 8) & 0xFF).to(torch.uint8)
    cab[:, :, 2], cab[:, :, 3] = (q[:, 1::2] & 0xFF).to(torch.uint8), ((q[:, 1::2] >> 8) & 0xFF).to(torch.uint8)
    cab[:, :, 4] = ((q[:, 0::2] >> 16) | ((q[:, 1::2] >> 16) << 4)).to(torch.uint8)
    fields = (torch.arange(P) * 53) % 23040
    seal(0x86, caps[:, 0], fields)
    seal(0x86, caps[:, 1], (fields + 20) % 23040)
    return caps, L


def ud_merge_positions(cases):
    caps, _ = cases
    return ud_smoothing_model(caps[:, 0].numpy(), np.zeros(caps.shape[0], np.int64))[1]


def _ud_raw_np(cap, pos):
    cab = 10 + 5 * (pos >> 1)
    hi = cap[:, cab + 4].astype(np.int64)
    qds = (cap[:, cab + 2 * (pos & 1)].astype(np.int64) | (cap[:, cab + 1 + 2 * (pos & 1)].astype(np.int64) << 8) |
           (((hi >> 4) if pos & 1 else (hi & 0xF)) << 16))
    return qds


def ud_decode_model(qds, base3=24567, mask_fault=False):
    """ud_decode's branchless form: (dist before smoothing, scale, quality)."""
    scale = qds & 3
    packed = (base3 << 45) | (8187 << 30) | (2046 << 15)
    base = (packed >> (15 * scale)) & 0x7FFF
    quality = ((qds >> (12 + scale)) << scale) & 0xFF
    mask = (0x1000 << scale) - (8 if mask_fault else 4)
    return (qds & mask) * (scale + 2) + (base << 2), scale, quality


def ud_decode_sdk(qds):
    t = torch.from_numpy(qds)
    cap = torch.zeros(t.numel(), 170, dtype=torch.uint8)
    cap[:, 10], cap[:, 11], cap[:, 14] = (t & 0xFF).to(torch.uint8), ((t >> 8) & 0xFF).to(torch.uint8), (t >> 16).to(torch.uint8)
    d, s, q = ultra_dense_sample(cap, 0)
    return d.numpy(), s.numpy(), q.numpy()


def ud_smoothing_model(cap, last_in, spread=4):
    """The kernel's smoothing chain for one capsule: the nine candidates of the first sample (r0 - 4 .. r0 + 4 when it
    is scale 0), run until they merge (ud_pm), then the table lookup apply() for the real input, then the replay of
    the positions before ud_pm.  Returns (smoothed scale-0 distances [P, 64], ud_pm [P], last out [P])."""
    P = cap.shape[0]
    raws = [ud_decode_model(_ud_raw_np(cap, pos))[:2] for pos in range(64)]
    r0, sc0 = raws[0]
    cand = [np.where(sc0 == 0, r0 - spread + k, r0) for k in range(9)]
    merged = sc0 != 0
    pm = np.where(merged, 0, 64)
    for pos in range(1, 64):
        r, sc = raws[pos]
        for k in range(9):
            c = cand[k]
            cand[k] = np.where((sc == 0) & (c != 0) & (np.abs(r - c) <= 8), (r + c) >> 1, r)
        now = ~merged & np.all([cand[k] == cand[0] for k in range(9)], axis=0)
        pm = np.where(now, pos, pm)
        merged |= now
    # outcome for the real input: the candidate index the first sample's smoothing lands on
    k = np.full(P, 4)
    near = (sc0 == 0) & (last_in != 0) & (np.abs(r0 - last_in) <= 8)
    k = np.where(near, ((r0 + last_in) >> 1) - (r0 - 4), k)
    k = np.clip(k, 0, 8)
    outs = np.stack(cand, 1)
    last_out = np.where(merged, outs[:, 0], outs[np.arange(P), k])
    # the smoothed distances: replay from the real input (the kernel replays positions < ud_pm; after it every
    # candidate agrees, so the plain recurrence gives the same values)
    dist = np.zeros((P, 64), np.int64)
    last = last_in.copy()
    for pos in range(64):
        r, sc = raws[pos]
        last = np.where((sc == 0) & (last != 0) & (np.abs(r - last) <= 8), (r + last) >> 1, r)
        dist[:, pos] = last
    return dist, pm, last_out


def check_smoothing(model):
    """The sweep's checker for the smoothing chain: the last distance a capsule leaves, from the kernel's tables,
    against the SDK's recurrence, over every smoothing case."""
    caps, last_in = smoothing_cases()
    _, _, _, _, want = sdk_pairs(0x86, caps[:, 0], caps[:, 1], torch.zeros_like(last_in), last_in)
    _, _, got = model(caps[:, 0].numpy(), last_in.numpy())
    return int((got != want.numpy()).sum())


# ---- numpy models of the kernel's other formulations, and their checkers ---------------------------------------------
def varbitscale_sel_model(s, nibbles=0x4443333332211100, srcs=0xD00700500200000):
    l = (nibbles >> (4 * (s >> 8))) & 0xF
    src = (srcs >> (12 * l)) & 0xFFF
    dst = np.where(l != 0, 512, 0) << ((0x53200 >> (4 * l)) & 0xF)
    return dst + ((s - src) << l), l


def check_varbitscale(model):
    """Every 12-bit code of the cabin-code family: value and level against the SDK's loop."""
    s = np.arange(4096, dtype=np.int64)
    v, l = model(s)
    wv, wl = varbitscale_decode(torch.from_numpy(s))
    return int(((v != wv.numpy()) | (l != wl.numpy())).sum())


def check_ud_decode(model):
    """Every 20-bit qds of the sample-code family against the SDK's switch."""
    q = np.arange(1 << 20, dtype=np.int64)
    d, s, qu = model(q)
    wd, ws, wq = ud_decode_sdk(q)
    return int(((d != wd) | (s != ws) | (qu != wq)).sum())


@functools.lru_cache(maxsize=None)
def _angle_sample(k=400000):
    p, d = angle_cases()
    rng = np.random.default_rng(1)
    i = rng.choice(p.numel(), k, replace=False)
    edge = np.flatnonzero((d.numpy() < 0) | (d.numpy() == 0))[:20000]
    cur0 = np.flatnonzero(np.fmod(p.numpy() + d.numpy(), FULL_Q8) < 64 * 4)[::7][:20000]  # wraps on the last sample
    i = np.concatenate([i, edge, cur0])
    return p.numpy()[i], d.numpy()[i]


def check_express_sync(model):
    p, d = _angle_sample()
    got, want = model(p, d), express_sync_sdk(p, d)
    return int(sum((g != w).sum() for g, w in zip(got, want)))


def check_raw_sync(model):
    p, d = _angle_sample()
    bad = 0
    for n in (40, 64):
        inc = c_div(d << 8, n)
        got, _ = model(p, inc, n)
        want = raw_sync_sdk(p, inc, n)
        bad += int(sum((g != w).sum() for g, w in zip(got, want)))
    return bad


def xor_fold_model(caps, cb, fold16=True, first_shift=True):
    """The kernel's checksum: 32-bit words folded (84 / 132 bytes), 16-bit halves (170 bytes), then the two bytes."""
    if cb % 4 == 0:
        w = caps[:, :cb].copy().view("<u4").astype(np.int64)
        x = (w[:, 0] >> 16) if first_shift else w[:, 0]
        for k in range(1, cb // 4):
            x = x ^ w[:, k]
        if fold16:
            x ^= x >> 16
    else:
        h = caps[:, :cb].copy().view("<u2").astype(np.int64)
        x = np.zeros(caps.shape[0], np.int64)
        for k in range(1, cb // 2):
            x ^= h[:, k]
    return (x ^ (x >> 8)) & 0xFF


def check_xor(model):
    bad = 0
    for ans in XOR_FORMATS:
        caps = checksum_pairs(ans)[:, 1]
        want = _xor_reduce(caps[:, 2:].long())
        bad += int((model(caps.numpy(), CB[ans]) != want.numpy()).sum())
    return bad


def test_kernel_models_pass_their_checkers():
    assert check_varbitscale(varbitscale_sel_model) == 0
    assert check_ud_decode(ud_decode_model) == 0
    assert check_express_sync(express_sync_model) == 0
    assert check_raw_sync(raw_sync_mask_model) == 0
    assert check_xor(xor_fold_model) == 0
    assert check_smoothing(ud_smoothing_model) == 0


MUTANTS = {
    "varbitscale nibble 0x4443333332211100 -> 0x4443333332221100": (
        check_varbitscale, lambda s: varbitscale_sel_model(s, nibbles=0x4443333332221100)),
    "varbitscale source base 0x500 -> 0x4FF": (
        check_varbitscale, lambda s: varbitscale_sel_model(s, srcs=0xD007004FF200000)),
    "ud_decode scale-3 base 24566": (check_ud_decode, lambda q: ud_decode_model(q, base3=24566)),
    "ud_decode field mask - 8": (check_ud_decode, lambda q: ud_decode_model(q, mask_fault=True)),
    "express remainder rem > kFull": (check_express_sync, lambda p, d: express_sync_model(p, d, strict_sub=True)),
    "raw_sync_mask early exit with <=": (check_raw_sync, lambda p, i, n: raw_sync_mask_model(p, i, n, exit_le=True)),
    "raw_sync_mask remainder rem > kFull": (check_raw_sync, lambda p, i, n: raw_sync_mask_model(p, i, n, strict_sub=True)),
    "xor fold without x ^= x >> 16": (check_xor, lambda c, cb: xor_fold_model(c, cb, fold16=False)),
    "xor fold without w[0] >> 16": (check_xor, lambda c, cb: xor_fold_model(c, cb, first_shift=False)),
    "smoothing candidates over +-3": (check_smoothing, lambda c, l: ud_smoothing_model(c, l, spread=3)),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_planted_faults_are_rejected(name):
    checker, model = MUTANTS[name]
    assert checker(model) > 0, name
