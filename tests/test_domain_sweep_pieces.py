"""The pieces of the domain sweeps (tests/test_gpu_domain_sweeps.py), checked without a GPU.

The scan kernels take arithmetic shortcuts that the parity suite's random scans seldom reach: mode_a_bin_fast
(rpl_device.cuh) bins a Mode A key by an integer quotient and falls back to the reference's float chain only for keys
close to a bin edge, and dist_to_m divides by 4000 with a reciprocal refinement.  The GPU sweeps run every key
through every Mode A bin edge of thousands of beam counts, and every distinct distance through Mode B, and compare
with expectations computed here:

  * the Mode A bins of every key by the reference's float chain (rplidar_node.cpp:586-652), restated in numpy, with
    no use of the oracle or of the device shortcut;
  * bin covers: for a beam count M, scans of exactly M measured nodes on distinct keys, one node in every bin, such
    that max_b w_b scans (w_b = keys in bin b) put every key into its bin at least once; each key carries its own
    distance (4 * key + 4) and quality, so an output bin shows which key landed in it;
  * tie scans: the two end keys of half the bins on one distance with different qualities, the other bins empty
    (the reference's stable ascending-angle order and strict '<' make the lower key win, in both orientations);
  * one checker for all of it, which runs on CPU tensors here and on device tensors in the GPU file.

The checker is shown to have power: fed a numpy model of mode_a_bin_fast with a wrong guard width, without its float
fall-back, with key 0 of inverted scans sent through the integer quotient or with M - 1 passed for M, it reports a
mismatch; fed the unmutated model, none.
"""
import numpy as np
import pytest
import torch

F32 = np.float32
TWO_PI = 2.0 * np.pi  # the reference's 2.0 * M_PI, a double
KEYS = 65536          # angle_z_q14 is a u16
MODE_A_MAP_MAX = 32768  # scan_tma.cu: the ring kernel's Mode A index map holds this many points

# ---- the beam counts the sweeps run ----------------------------------------------------------------------------------
_rng = np.random.default_rng(20261016)
SMALL_MS = list(range(1, 8193))  # the shared-memory kernel: every stride it serves
RING_MS = sorted(set(range(1, 1537)) | set(range(1537, 8193, 7)) | set(range(8190, 8201)) | set(range(16380, 16391))
                 | set(range(32760, 32769)) | set(int(m) for m in _rng.integers(1537, MODE_A_MAP_MAX + 1, 300)))
# above 65239 the float chain leaves some bins without a key (two keys share the neighbouring bin): 65255, 65535 and
# 65536 are among those, and a scan of M measured nodes then has to put two of them into one bin
WIDE_MS = sorted(set(RING_MS) | set(int(m) for m in _rng.integers(MODE_A_MAP_MAX + 1, KEYS + 1, 100))
                 | {65255, 65535, KEYS})
del _rng


# ---- 1. the reference's float chain ----------------------------------------------------------------------------------
def _angles():
    """angle_rad of every key (float32), and the inverted angle 2*pi - angle_rad with the reference's wrap."""
    k = np.arange(KEYS, dtype=F32)
    deg = (k * F32(90.0)) / F32(16384.0)                              # getAngle: exact
    rad = (deg.astype(np.float64) * (np.pi / 180.0)).astype(F32)     # double product rounded to float
    inv = (TWO_PI - rad.astype(np.float64)).astype(F32)
    wrap = inv.astype(np.float64) >= TWO_PI
    inv = np.where(wrap, (inv.astype(np.float64) - TWO_PI).astype(F32), inv)
    return rad, inv


_RAD, _RAD_INV = _angles()


def mode_a_increment(m):
    """LaserScan.angle_increment of Mode A: float(2*pi / M), the division in double."""
    return F32(TWO_PI / float(m))


def mode_b_increment(m):
    return F32(TWO_PI / float(m - 1 if m > 1 else 1))


def float_chain_bins(m, inverted):
    """The Mode A bin of every key: (int)(angle / angle_increment), the quotient in float."""
    a = _RAD_INV if inverted else _RAD
    return ((a - F32(0.0)) / mode_a_increment(m)).astype(np.int64)


def scan_order(inverted):
    """The keys in the order their bins ascend: ascending, or inverted key 0 (wrapped to bin 0) then descending."""
    return np.concatenate([[0], np.arange(KEYS - 1, 0, -1)]) if inverted else np.arange(KEYS)


# ---- 2. bin covers and tie scans ---------------------------------------------------------------------------------
def node_dist(key):
    return 4 * key + 4


def node_quality(key):
    return (key * 97 + (key >> 8)) & 0xFF


TIE_QUALITY_FLIP = 0xA4  # changes the quality in both protocols (new: all 8 bits, old: bits 2..7)


class Cover:
    """The float chain's bins of one (M, orientation), as the builders need them: keys grouped by bin in scan order
    (grouped[start[b]:start[b] + width[b]] are bin b's keys), and for every bin the float chain leaves empty one bin
    with two or more keys (extra) that takes a second node, so that a scan has M measured nodes."""

    def __init__(self, m, inverted):
        self.m, self.inverted = m, bool(inverted)
        self.bins = float_chain_bins(m, inverted)
        order = scan_order(inverted)
        self.grouped = order[np.argsort(self.bins[order], kind="stable")]
        self.width = np.bincount(self.bins, minlength=m)
        assert len(self.width) == m, (m, inverted, "a key binned at or past M")
        self.start = np.cumsum(self.width) - self.width
        self.nonempty = np.flatnonzero(self.width)
        n_empty = m - len(self.nonempty)
        wide = np.flatnonzero(self.width >= 2)
        self.extra = wide[np.linspace(0, len(wide) - 1, n_empty).astype(np.int64)] if n_empty else wide[:0]
        assert len(np.unique(self.extra)) == n_empty
        self.n_scans = int(self.width.max())

    def tensors(self, dev):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(dev)
        return t(self.grouped), t(self.start), t(self.width), t(self.nonempty), t(self.extra)


def cover_scans(cov, dev="cpu"):
    """(keys [W, M], winner [W, M]): the node keys of the W = max_b w_b scans of a cover (scan j gives bin b its
    key number j mod w_b, and an extra bin also key number j + 1 mod w_b), and for every bin the key whose node must
    land there (-1: none).  Distances grow with the key, so the lower key of a bin with two nodes wins."""
    grouped, start, width, nonempty, extra = cov.tensors(dev)
    j = torch.arange(cov.n_scans, device=dev)[:, None]
    w = width.clamp(min=1)
    prim = grouped[start[None, :] + j % w[None, :]]                       # [W, M], by bin
    prim = torch.where(width[None, :] > 0, prim, torch.full_like(prim, -1))
    ext = grouped[start[extra][None, :] + (j + 1) % w[extra][None, :]]   # [W, E]
    keys = torch.cat([prim[:, nonempty], ext], 1)
    winner = prim.clone()
    winner[:, extra] = torch.minimum(prim[:, extra], ext)
    return keys, winner


def tie_scan(cov, dev="cpu"):
    """(keys, dist, quality, winner) of one scan, each [1, M]: in M // 2 bins of two or more keys (every second bin
    first) the first and the last key of the bin on one distance, the lower key's, with different qualities; for an
    odd M one more bin with a single node; every other bin empty.  The lower key must win: the reference visits the
    points in ascending angle order and replaces a bin's value only on a strictly smaller distance."""
    m = cov.m
    wide = np.flatnonzero(cov.width >= 2)
    pick = np.concatenate([wide[wide % 2 == 0], wide[wide % 2 == 1]])[: m // 2]
    assert len(pick) == m // 2, (m, cov.inverted)
    first, last = cov.grouped[cov.start[pick]], cov.grouped[cov.start[pick] + cov.width[pick] - 1]
    lo, hi = np.minimum(first, last), np.maximum(first, last)
    keys, dist, qual = [lo, hi], [node_dist(lo), node_dist(lo)], [node_quality(lo), node_quality(lo) ^ TIE_QUALITY_FLIP]
    winner = np.full(m, -1, np.int64)
    winner[pick] = lo
    if m % 2:
        single = np.setdiff1d(cov.nonempty, pick)[0]
        k = cov.grouped[cov.start[single]:cov.start[single] + 1]
        keys, dist, qual = keys + [k], dist + [node_dist(k)], qual + [node_quality(k)]
        winner[single] = k[0]
    t = lambda parts: torch.from_numpy(np.concatenate(parts).astype(np.int64)[None]).to(dev)
    return t(keys), t(dist), t(qual), torch.from_numpy(winner[None]).to(dev)


def pack_nodes(keys, dist, qual):
    """int64 words of rpl_node_hq {u16 angle_z_q14, u32 dist_mm_q2, u8 quality, u8 flag = 0}, little-endian."""
    x = keys | ((dist & 0xFFFF) << 16)
    y = (dist >> 16) | (qual << 16)
    return x | (y << 32)


def rolled(a, seed):
    """Each row rotated by its own amount (the revolution starts anywhere in the buffer); a [S, n]."""
    S, n = a.shape
    r = (torch.arange(S, device=a.device)[:, None] * 7919 + seed) % max(n, 1)
    return a.gather(1, (torch.arange(n, device=a.device)[None, :] + r) % max(n, 1))


# ---- expectations: float32(dist) / 4000 and the intensity of each key --------------------------------------------------
def _bits(a):
    return torch.from_numpy(np.ascontiguousarray(a, F32).view(np.int32).astype(np.int64))


_KEY = np.arange(KEYS, dtype=np.int64)
RANGE_BITS = _bits(node_dist(_KEY).astype(F32) / F32(4000.0))  # ascending in the key (positive floats)
INTEN_BITS = {1: _bits(node_quality(_KEY).astype(F32)), 0: _bits((node_quality(_KEY) >> 2).astype(F32))}
INF_BITS = int(np.array(np.inf, F32).view(np.int32))


class Tables:
    """The expectation tables on one device."""

    def __init__(self, dev):
        self.range = RANGE_BITS.to(dev)
        self.inten = {p: v.to(dev) for p, v in INTEN_BITS.items()}


def first_mode_a_mismatch(ranges, intens, winner, ms, newp, tab):
    """(scan, bin) of the first LaserScan slot that differs from what the winner keys say, bit for bit -- ranges
    float32(dist) / 4000 and the protocol's intensity of the winning key, +inf and 0 for an empty bin -- or that was
    written at or behind beam_count (ranges and intensities must still hold their NaN pre-fill there); None if every
    slot is right.  ranges, intens: float32 [S, stride]; winner: int64 [S, >= M]; ms: int64 [S]."""
    S, stride = ranges.shape
    col = torch.arange(stride, device=ranges.device)[None, :]
    live = col < ms[:, None]
    w = torch.full((S, stride), -1, dtype=torch.int64, device=ranges.device)
    w[:, : winner.shape[1]] = winner
    w = torch.where(live, w, torch.full_like(w, -1))
    hit = w >= 0
    wk = w.clamp(min=0)
    exp_r = torch.where(hit, tab.range[wk], torch.full_like(wk, INF_BITS))
    exp_i = torch.where(hit, tab.inten[newp][wk], torch.zeros_like(wk))
    got_r, got_i = ranges.view(torch.int32).to(torch.int64), intens.view(torch.int32).to(torch.int64)
    ok = torch.where(live, (got_r == exp_r) & (got_i == exp_i), torch.isnan(ranges) & torch.isnan(intens))
    if bool(ok.all()):
        return None
    bad = (~ok).nonzero()[0]
    return int(bad[0]), int(bad[1])


def landed_key(range_bits, tab):
    """The key whose distance converts to these range bits (None for +inf / anything else)."""
    r = tab.range
    i = int(torch.searchsorted(r, torch.tensor([range_bits], device=r.device)))
    return i if i < KEYS and int(r[i]) == range_bits else None


def describe_mode_a_mismatch(where, ranges, winner, ms, inverted, kernel, tab):
    s, b = where
    m = int(ms[s])
    want = int(winner[s, b]) if b < winner.shape[1] else -1
    got = int(ranges[s, b].view(torch.int32))
    if b >= m:
        return f"{kernel}: M={m} {'inverted' if inverted else 'upright'}: slot {b} behind beam_count was written"
    return (f"{kernel}: M={m} {'inverted' if inverted else 'upright'}: bin {b} expected key "
            f"{want if want >= 0 else 'none (empty bin)'}, got the range of key {landed_key(got, tab)} "
            f"(bits {got:#010x}) -- or the right key with the wrong intensity")


# ---- 3. numpy models of mode_a_bin_fast, with the faults the sweep must see ---------------------------------------------
def model_bins(keys, m, inverted, guard=lambda m: (m >> 5) + 2, fallback=True, key0_exception=True, key0_integer=False,
               m_passed=None):
    """mode_a_bin_fast(key, m, inc, inverted) in numpy (u32 arithmetic), the float chain being float_chain_bins of
    the true M (the kernels compute inc from the beam count).  key0_exception=False drops the explicit exception for
    key 0 of inverted scans; key0_integer=True sends that key through the integer quotient whatever the guard says."""
    mi = m if m_passed is None else m_passed
    keys = np.asarray(keys, np.int64)
    kk = (KEYS - keys) if inverted else keys
    t = (kk * mi) & 0xFFFFFFFF
    frac = t & 0xFFFF
    g = guard(mi)
    fast = ((frac - g) & 0xFFFFFFFF) <= ((KEYS - 2 * g) & 0xFFFFFFFF)
    if inverted and key0_exception:
        fast &= keys != 0
    if not fallback:
        fast[:] = True
    if inverted and key0_integer:
        fast |= keys == 0
    return np.where(fast, t >> 16, float_chain_bins(m, inverted)[keys])


MUTANTS = {
    "guard m >> 6": dict(guard=lambda m: m >> 6),
    "no float fall-back": dict(fallback=False),
    "inverted key 0 through the integer quotient": dict(key0_integer=True),
    "M - 1 passed for M": dict(m_passed="m-1"),
}


def simulate_mode_a(keys, m, inverted, newp, **fault):
    """What a scatter-min Mode A kernel binning with model_bins writes for cover scans (keys [S, M]): per bin the
    node with the smallest distance (here the smallest key), +inf and 0 where nothing fell; a bin at or past M is
    dropped, as the reference's bounds check does."""
    if fault.get("m_passed") == "m-1":
        fault = dict(fault, m_passed=max(m - 1, 1))
    S = keys.shape[0]
    b = torch.from_numpy(model_bins(keys.numpy(), m, inverted, **fault))
    keep = (b >= 0) & (b < m)
    big = torch.full((S, m + 1), KEYS, dtype=torch.int64)
    big.scatter_reduce_(1, torch.where(keep, b, torch.full_like(b, m)), keys, reduce="amin")
    win = big[:, :m]
    hit = win < KEYS
    wk = win.clamp(max=KEYS - 1)
    r = torch.where(hit, RANGE_BITS[wk], torch.full_like(wk, INF_BITS)).to(torch.int32).view(torch.float32)
    i = torch.where(hit, INTEN_BITS[newp][wk], torch.zeros_like(wk)).to(torch.int32).view(torch.float32)
    return r, i


def model_sweep_mismatch(ms, **fault):
    """The first (M, orientation, scan, bin) over the cover scans of ms where the checker rejects the model's output."""
    tab = Tables("cpu")
    for m in ms:
        for inverted in (False, True):
            cov = Cover(m, inverted)
            keys, winner = cover_scans(cov)
            newp = (m + inverted) & 1
            r, i = simulate_mode_a(keys, m, inverted, newp, **fault)
            bad = first_mode_a_mismatch(r, i, winner, torch.full((keys.shape[0],), m), newp, tab)
            if bad is not None:
                return m, inverted, bad
    return None


# ---- the CPU tests ---------------------------------------------------------------------------------------------------
def test_float_chain_bins_are_monotone_and_in_range_over_the_swept_beam_counts():
    """Every bin the sweeps expect lies in [0, M), and bins never descend along the scan order: the ring kernel's
    head/tail/gap logic relies on it, and it makes each bin's keys one run of that order."""
    for m in sorted(set(SMALL_MS) | set(WIDE_MS)):
        for inverted in (False, True):
            b = float_chain_bins(m, inverted)
            assert b.min() >= 0 and b.max() < m, (m, inverted)
            assert (np.diff(b[scan_order(inverted)]) >= 0).all(), (m, inverted)
    assert float_chain_bins(7, True)[0] == 0  # inverted key 0 wraps to 1.7e-7 rad


BUILDER_MS = sorted(set(range(1, 65)) | set(range(65, KEYS + 1, 97)) | {1536, 8191, 8192, 32767, 32768, 65254, 65255,
                                                                          65535, KEYS})


@pytest.mark.parametrize("inverted", [False, True])
def test_cover_scans_put_every_key_into_its_bin(inverted):
    n_empty_ms = 0
    for m in BUILDER_MS:
        cov = Cover(m, inverted)
        keys, winner = cover_scans(cov)
        k, w = keys.numpy(), winner.numpy()
        W = cov.n_scans
        assert k.shape == (W, m) and w.shape == (W, m)
        assert W == cov.width.max() and W <= -(-KEYS // m) + 2, (m, W)
        srt = np.sort(k, 1)
        assert (srt >= 0).all() and (np.diff(srt, axis=1) > 0).all(), (m, "a key twice in one scan")
        count = np.bincount(k.ravel(), minlength=KEYS)
        assert (count >= 1).all(), (m, "a key no scan carries")
        # key number i of bin b appears in the scans j = i mod w_b (+ the extra ones): no key more often than that
        bins = cov.bins
        assert (count <= -(-W // cov.width[bins]) + 1).all()
        # one node per bin: every bin with keys gets one, an empty one none, and the extra bins two
        b_of = bins[k]
        per_bin = np.stack([np.bincount(row, minlength=m) for row in b_of])
        want = (cov.width > 0).astype(np.int64)
        want[cov.extra] += 1
        assert (per_bin == want[None, :]).all(), m
        assert (bins[np.where(w >= 0, w, 0)] == np.arange(m)[None, :])[w >= 0].all()
        assert ((w >= 0) == (cov.width > 0)[None, :]).all()
        n_empty_ms += len(cov.extra) > 0
        if not len(cov.extra):
            assert (np.sort(w, 1) == srt).all()  # exactly one node per bin: the winners are the nodes
    assert n_empty_ms >= 2  # beam counts where the float chain leaves a bin empty are among them


@pytest.mark.parametrize("inverted", [False, True])
def test_tie_scans_share_half_the_bins(inverted):
    for m in [x for x in BUILDER_MS if x <= MODE_A_MAP_MAX]:
        cov = Cover(m, inverted)
        keys, dist, qual, winner = (t.numpy()[0] for t in tie_scan(cov))
        assert len(keys) == m and len(np.unique(keys)) == m
        b = cov.bins[keys]
        per_bin = np.bincount(b, minlength=m)
        assert (per_bin <= 2).all() and (per_bin == 2).sum() == m // 2 and (per_bin == 1).sum() == m % 2
        o = np.lexsort((keys, b))  # the nodes by bin, then key
        shared = per_bin[b[o]] == 2
        lo, hi = o[shared][0::2], o[shared][1::2]  # the lower and the higher key of each shared bin
        assert (b[lo] == b[hi]).all() and (dist[lo] == dist[hi]).all() and (dist[lo] == node_dist(keys[lo])).all()
        assert (qual[lo] == node_quality(keys[lo])).all() and ((qual[lo] >> 2) != (qual[hi] >> 2)).all()
        assert (winner[b[lo]] == keys[lo]).all()
        assert ((winner >= 0) == (per_bin > 0)).all()


def test_checker_passes_the_float_chain_and_the_unmutated_model():
    tab = Tables("cpu")
    for m in (1, 2, 3, 7, 360, 3200, 65255, KEYS):
        for inverted in (False, True):
            keys, winner = cover_scans(Cover(m, inverted))
            S = keys.shape[0]
            ms = torch.full((S,), m)
            # a perfect kernel: the winners' values, NaN behind M
            wk = winner.clamp(min=0)
            r = torch.where(winner >= 0, RANGE_BITS[wk], torch.full_like(wk, INF_BITS)).to(torch.int32).view(torch.float32)
            i = torch.where(winner >= 0, INTEN_BITS[1][wk], torch.zeros_like(wk)).to(torch.int32).view(torch.float32)
            pad = torch.full((S, 3), float("nan"))
            r, i = torch.cat([r, pad], 1), torch.cat([i, pad], 1)
            assert first_mode_a_mismatch(r, i, winner, ms, 1, tab) is None
            # ... and it notices a slot written behind M, a swapped pair of bins, a wrong intensity protocol
            bad = r.clone()
            bad[0, m] = 1.0
            assert first_mode_a_mismatch(bad, i, winner, ms, 1, tab) == (0, m)
            if m >= 2:
                bad = r.clone()
                bad[S - 1, [0, 1]] = bad[S - 1, [1, 0]]
                assert first_mode_a_mismatch(bad, i, winner, ms, 1, tab) == (S - 1, 0)
            assert first_mode_a_mismatch(r, i, winner, ms, 0, tab) is not None
    ms = sorted(set(range(1, 200)) | set(RING_MS[::17]) | set(WIDE_MS[-12:]))
    assert model_sweep_mismatch(ms) is None


@pytest.mark.parametrize("fault", list(MUTANTS))
def test_checker_rejects_a_faulty_mode_a_bin_fast(fault):
    """Each fault of mode_a_bin_fast is seen by the cover scans of the swept beam counts."""
    found = model_sweep_mismatch(sorted(set(SMALL_MS) | set(WIDE_MS)), **MUTANTS[fault])
    assert found is not None, f"the sweep cannot see the fault: {fault}"


def test_inverted_key0_exception_is_covered_by_the_guard():
    """mode_a_bin_fast's explicit exception for key 0 of inverted scans never decides a bin: (65536 - 0) * M has no
    fractional part, and the edge guard sends such a key to the float chain anyway.  Dropping the exception alone is
    no fault; the fault it guards against -- key 0 through the integer quotient, bin M -- is rejected above."""
    k = np.arange(KEYS)
    for m in sorted(set(WIDE_MS) | set(range(1, 300))):
        assert (model_bins(k, m, True) == model_bins(k, m, True, key0_exception=False)).all(), m
