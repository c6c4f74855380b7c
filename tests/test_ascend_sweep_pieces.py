"""The pieces of the angle-compensation sweeps (tests/test_gpu_ascend_sweeps.py), checked without a GPU.

ascendScanData_ (reference src/sdk/src/sl_lidar_driver.cpp:129-184) walks back from the first measured node to give
node 0 an angle (head tune: each step getAngle(next) - 360.f/count, clamped at 0 and re-quantised), then gives every
other unmeasured node i frontAngle + i * inc (minus 360 when the sum is > 360.0f), and sorts the nodes by angle.  The
kernels copy that float arithmetic (ascend_step, ascend_fill_key, ascend_head_key in rpl_device.cuh).  What the GPU
sweeps need is built and checked here:

  * the restatement: the reference's code in numpy float32, vectorised over scans -- the head chain through the
    map g_n(k) = key(max(0, deg(k) - step)) over the whole key space, every fill key of a scan at once, then the
    (u16)(u32) store and a stable sort by final key (the project's tie rule); pinned against the reference's own
    ascendScanData (recorded in tests/golden/reference_outputs.npz where oracle/_ref is not built) and against
    oracle/scan_oracle.cpp;
  * the case builders: n, the first measured node f with its key K, and extra measured nodes placed on computed
    final keys -- they reach the fill angles that round to exactly 360.0f (stored as key 0), the wrap, the head clamp
    at exactly f steps and short of it, and 0..17 shared final keys in every position the shared-memory kernel's
    duplicate path distinguishes;
  * one checker, written in torch so that it runs on numpy arrays (as CPU tensors) and on device tensors: the torch
    restatement divides by 90 through a tensor, since tensor / python_scalar multiplies by the reciprocal.

The checker is shown to have power: numpy models of six faults of the arithmetic are each rejected, and the
unmutated model passes.  Two more variants are shown to be no fault at all, so that no sweep can reject them: the wrap
tested with >= 360 (at exactly 360.0f both branches store key 0), and the wrap applied after quantising (for every
float in (360, 720) the u16 store of the quotient gives the key of the angle minus 360).
"""
import functools

import numpy as np
import pytest
import torch

from reference_outputs import Reference, same

F32 = np.float32
KEYS = 65536
OK, FAIL = 0, 0x80008001
SENTINEL = 0x5A5A5A5A5A5A5A5A  # what every output slot holds before a launch
SHARED_NS = (2, 3, 4, 8, 12, 360, 720, 1000, 3200, 4096, 8191, 8192)  # every key through these
WIDE_NS = (8193, 16384, 32768, 65536)
CHAIN_NS = tuple(range(2, 65)) + (360, 3200, 8192)  # every first measured index through these
MAX_DUP = 17  # shared final keys the builders reach: the shared-memory kernel resolves 16, hands on 17
_SPREAD = 2 ** 17  # sort key = final key * _SPREAD + buffer position


# ---- 1. the restatement (numpy float32) ------------------------------------------------------------------------------
def key_deg(k):
    """getAngle: angle_z_q14 * 90.f / 16384.f"""
    return (np.asarray(k).astype(F32) * F32(90.0)) / F32(16384.0)


def deg_key(v):
    """setAngle: angle_z_q14 = sl_u32(v * 16384.f / 90.f), stored in a u16"""
    return ((np.asarray(v, F32) * F32(16384.0)) / F32(90.0)).astype(np.int64) & 0xFFFF


def step_of(n):
    """inc_origin_angle = 360.f / count"""
    return F32(360.0) / np.asarray(n).astype(F32)


def fill_keys(front_deg, i, step, ge=False, fma=False, wrap_after=False):
    """The key an unmeasured node i >= 1 gets: frontAngle + i * inc, minus 360 when > 360.0f.  Faults: ge (>= 360),
    fma (the sum rounded once), wrap_after (no subtraction: the u16 store wraps the quotient)."""
    front_deg, step = np.asarray(front_deg, F32), np.asarray(step, F32)
    if fma:
        a = (front_deg.astype(np.float64) + np.asarray(i, np.float64) * step.astype(np.float64)).astype(F32)
    else:
        a = front_deg + np.asarray(i).astype(F32) * step
    if wrap_after:
        return deg_key(a)
    wrap = (a >= F32(360.0)) if ge else (a > F32(360.0))
    return deg_key(np.where(wrap, a - F32(360.0), a))


@functools.lru_cache(maxsize=None)
def chain_map(n):
    """g_n: one head-tune step from every key"""
    return deg_key(np.maximum(key_deg(np.arange(KEYS)) - step_of(n), F32(0.0)))


def chain_power(n, f):
    """g_n^f over every key: node 0's key when the first measured node is f with key K is chain_power(n, f)[K]"""
    out, p = np.arange(KEYS), chain_map(n)
    while f:
        if f & 1:
            out = p[out]
        p, f = p[p], f >> 1
    return out


@functools.lru_cache(maxsize=None)
def clamp_steps(n):
    """For every key, the steps the head chain takes to reach key 0 (g_n(k) < k for k > 0)"""
    g = chain_map(n).tolist()
    c = [0] * KEYS
    for k in range(1, KEYS):
        c[k] = c[g[k]] + 1
    return np.array(c)


def head_keys(K, f, step, mode="walk", short=0):
    """Node 0's key for first measured keys K at indices f (vectorised).  Faults: mode "once" (deg(K) - f*step
    quantised once, clamped), "fill" (node 0 given the fill formula from the first measured node: deg(K) - f*step,
    plus 360 below 0), short (the walk stops that many steps early)."""
    K, f, step = np.asarray(K, np.int64), np.asarray(f, np.int64), np.asarray(step, F32)
    if mode in ("once", "fill"):
        a = key_deg(K) - f.astype(F32) * step
        a = np.maximum(a, F32(0.0)) if mode == "once" else np.where(a < F32(0.0), a + F32(360.0), a)
        return np.where(f > 0, deg_key(a), K)
    k = K.copy()
    for t in range(int((f - short).max(initial=0))):
        act = (t < f - short) & (k != 0)
        if not act.any():
            break
        k = np.where(act, deg_key(np.maximum(key_deg(k) - step, F32(0.0))), k)
    return k


def ascend_words(words, counts, ge=False, fma=False, chain="walk", chain_short=0, step_n1=False, wrap_after=False,
                 reverse_ties=False):
    """ascendScanData_ over a batch: words int64 [S, W] (rpl_node_hq little-endian), counts [S].  Returns (status [S],
    ascended words [S, W], SENTINEL behind each count).  The keyword arguments plant the faults of the sweeps' models."""
    words, counts = np.asarray(words, np.int64), np.asarray(counts, np.int64)
    S, W = words.shape
    col = np.arange(W)[None, :]
    live = col < counts[:, None]
    meas = live & (((words >> 16) & 0xFFFFFFFF) != 0)
    anym = meas.any(1)
    f = np.where(anym, meas.argmax(1), 0)
    K = words[np.arange(S), f] & 0xFFFF
    step = step_of(np.maximum(counts - 1 if step_n1 else counts, 1))
    k0 = head_keys(K, f, step, chain, chain_short)
    fill = fill_keys(key_deg(k0)[:, None], col, step[:, None], ge, fma, wrap_after)
    final = np.where(meas, words & 0xFFFF, np.where(col == 0, k0[:, None], fill))
    tie = (W - 1 - col) if reverse_ties else col
    order = np.argsort(np.where(live, final * _SPREAD + tie, np.iinfo(np.int64).max), axis=1)
    out = np.take_along_axis((words & ~0xFFFF) | final, order, 1)
    out = np.where(anym[:, None], out, words)
    return np.where(anym, OK, FAIL), np.where(live, out, SENTINEL)


def ascend_nodes(nodes):
    """(sl_result, ascended copy) of one scan of NODE_DTYPE, by the restatement"""
    n = len(nodes)
    if n == 0:
        return FAIL, nodes.copy()
    st, out = ascend_words(np.ascontiguousarray(nodes).view(np.int64)[None], [n])
    return int(st[0]), out[0].view(nodes.dtype)


# ---- 2. the case builders --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def exact360(n):
    """(K, i) of every fill whose angle deg(K) + i * step rounds to exactly 360.0f (not > 360: stored as key 0)"""
    if n < 2:
        return np.zeros((0, 2), np.int64)
    i = np.arange(1, n)
    p = i.astype(F32) * step_of(n)
    k0 = np.floor((360.0 - p.astype(np.float64)) * (16384.0 / 90.0)).astype(np.int64)
    found = []
    for d in (-1, 0, 1, 2):
        k = k0 + d
        ok = (k >= 0) & (k < KEYS)
        kk = np.clip(k, 0, KEYS - 1)
        ok &= (key_deg(kk) + p) == F32(360.0)
        found.append(np.stack([kk[ok], i[ok]], 1))
    return np.unique(np.concatenate(found), axis=0)


def exact360_keys(n):
    return np.unique(exact360(n)[:, 0])


def spread(a, k):
    """at most k entries of a, evenly spaced (a power-of-two n has an exact-360 fill at every multiple of 65536 / n)"""
    return a if len(a) <= k else a[np.linspace(0, len(a) - 1, k).astype(np.int64)]


def node_dist(j):
    """the distance of a measured node at buffer position j: nonzero and distinct within a scan, so that no two Mode A
    points ever tie on a bin's minimum"""
    return 4 * np.asarray(j, np.int64) + 5


def junk(s, j):
    """(key, quality, flag) of the node at position j of scan s: an unmeasured node's key is overwritten, the other
    bytes must come through"""
    s, j = np.asarray(s, np.int64), np.asarray(j, np.int64)
    return (j * 40503 + s * 977 + 11) & 0xFFFF, (j * 13 + s * 7) & 0xFF, (j + s) & 3


class Cases:
    """Scans as (n, f, K) plus extra measured nodes (scan, position, key); f = -1: nothing measured."""

    def __init__(self, n, f, K, ex=None):
        self.n, self.f, self.K = (np.asarray(v, np.int64).ravel() for v in (n, f, K))
        self.f, self.K = np.broadcast_to(self.f, self.n.shape).copy(), np.broadcast_to(self.K, self.n.shape).copy()
        self.ex = np.zeros((0, 3), np.int64) if ex is None else np.asarray(ex, np.int64).reshape(-1, 3)

    def __len__(self):
        return len(self.n)

    @staticmethod
    def cat(parts):
        off, ex = 0, []
        for p in parts:
            ex.append(p.ex + [off, 0, 0])
            off += len(p)
        c = Cases(np.concatenate([p.n for p in parts]), np.concatenate([p.f for p in parts]),
                  np.concatenate([p.K for p in parts]))
        c.ex = np.concatenate(ex) if ex else c.ex
        return c

    def take(self, idx):
        idx = np.asarray(idx, np.int64)
        pos = np.full(len(self), -1)
        pos[idx] = np.arange(len(idx))
        keep = pos[self.ex[:, 0]] >= 0
        ex = self.ex[keep].copy()
        ex[:, 0] = pos[ex[:, 0]]
        c = Cases(self.n[idx], self.f[idx], self.K[idx], ex)
        return c

    def words(self, stride, dev=None, first_scan=0):
        """int64 words [S, stride] on `dev` (None: numpy); slots behind n are zero"""
        xp_t = dev is not None
        t = (lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)) if xp_t else np.asarray
        S = len(self)
        if xp_t:
            s = torch.arange(first_scan, first_scan + S, device=dev)[:, None]
            j = torch.arange(stride, device=dev)[None, :]
        else:
            s, j = np.arange(first_scan, first_scan + S)[:, None], np.arange(stride)[None, :]
        key, q, fl = junk(s, j) if not xp_t else ((j * 40503 + s * 977 + 11) & 0xFFFF, (j * 13 + s * 7) & 0xFF,
                                                   (j + s) & 3)
        w = key | (q << 48) | (fl << 56)
        meas = self.f >= 0
        rows = np.concatenate([np.flatnonzero(meas), self.ex[:, 0]])
        pos = np.concatenate([self.f[meas], self.ex[:, 1]])
        keys = np.concatenate([self.K[meas], self.ex[:, 2]])
        _, q0, f0 = junk(rows + first_scan, pos)
        val = keys | (node_dist(pos) << 16) | (q0 << 48) | (f0 << 56)
        w[t(rows), t(pos)] = t(val)
        live = j < t(self.n)[:, None]
        return w * live if not xp_t else torch.where(live, w, torch.zeros_like(w))


def fill_cases(n, keys):
    """family A: node 0 measured with key K, every other node unmeasured"""
    keys = np.asarray(keys, np.int64)
    return Cases(np.full(len(keys), n), 0, keys)


def front_keys_every_n(n, rng_seed=20261017):
    """family A's keys at every n: the ends and middle of the key space, n's exact-360 keys and three seeded keys"""
    rng = np.random.default_rng(rng_seed + n)
    return np.unique(np.concatenate([[0, 1, 16383, 32768, 65535], exact360_keys(n), rng.integers(0, KEYS, 3)]))


def clamp_edge_keys(n, f):
    """The keys either side of 'the chain clamps at exactly f steps': the smallest and largest key clamping at f,
    and their neighbours (clamping at f - 1 / f + 1)"""
    c = clamp_steps(n)
    at = np.flatnonzero(c == f)
    if not len(at):
        return np.zeros(0, np.int64)
    return np.unique(np.clip([at[0] - 1, at[0], at[-1], at[-1] + 1], 0, KEYS - 1))


@functools.lru_cache(maxsize=None)
def chain_cases(n, rng_seed=7):
    """family B: one measured node at every f in [0, n), keys 0, 1, the clamp edges of f, 65535, one seeded key"""
    rng = np.random.default_rng(rng_seed * 100003 + n)
    ns, fs, ks = [], [], []
    for f in range(n):
        k = np.unique(np.concatenate([[0, 1, KEYS - 1, int(rng.integers(0, KEYS))], clamp_edge_keys(n, f)]))
        ns.append(np.full(len(k), n))
        fs.append(np.full(len(k), f))
        ks.append(k)
    return Cases(np.concatenate(ns), np.concatenate(fs), np.concatenate(ks))


def chain_every_key_cases(n, every=1):
    """family B: every key (every `every`-th) at f in {1, 2, n/2, n - 1}"""
    k = np.arange(0, KEYS, every)
    fs = sorted({1, 2, n // 2, n - 1})
    return Cases(np.repeat(np.full(len(fs), n), len(k)), np.repeat(fs, len(k)), np.tile(k, len(fs)))


def final_keys_of(c, s):
    """final keys of scan s of c, by the restatement (before the sort)"""
    n, f, K = int(c.n[s]), int(c.f[s]), int(c.K[s])
    k0 = int(head_keys([K], [f], step_of(n))[0])
    fk = fill_keys(key_deg(k0), np.arange(n), step_of(n))
    fk[0] = k0
    fk[f] = K
    ex = c.ex[c.ex[:, 0] == s]
    fk[ex[:, 1]] = ex[:, 2]
    return fk


@functools.lru_cache(maxsize=None)
def shared_key_cases(seed=1):
    """family C: family A/B scans with measured nodes placed on computed final keys, for 0..17 shared final keys
    (extra nodes beyond the first of their key), the shared key from the fill, the head chain, the 360.0f fill (key 0),
    a clamped chain (key 0) and key 65535; up to four nodes on one key; the measured twin before and after the node it
    shares a key with; Mode A measured duplicates among them."""
    rng = np.random.default_rng(seed)
    scans = []  # (n, f, K, [(pos, key)])

    def add(n, f, K, targets=(), twins=(), on_key=None, count=1):
        """measured twins on the fill keys of `targets` (positions), placed at `twins` (positions); on_key: extra
        nodes on one explicit key"""
        c = Cases([n], [f], [K])
        fk = final_keys_of(c, 0)
        ex = [(int(j), int(fk[i])) for i, j in zip(targets, twins)]
        if on_key is not None:
            free = [j for j in range(f + 1, n) if j not in twins and j not in targets][:count]
            ex += [(j, on_key) for j in free]
        scans.append((n, f, K, ex))

    for n in (360, 1000, 3200, 8191, 8192):
        for d in range(MAX_DUP + 1):
            for v in range(2):
                f = 0 if v == 0 else int(rng.integers(1, 40))
                K = int(rng.integers(0, KEYS))
                pool = rng.permutation(np.arange(f + 1, n))[: 2 * d]
                targets, twins = pool[:d], pool[d:]
                add(n, f, K, targets, twins)
        # four nodes on one fill key (three twins), the twin before and after the node it shares
        K = int(rng.integers(0, KEYS))
        add(n, 0, K, [n // 2] * 3, [n // 2 - 5, n // 2 + 3, n - 1])
        # the shared key from the head chain (nonzero, f > 0) and node 0's twin at the end
        f = 30
        K = int(np.flatnonzero(clamp_steps(n) > f + 3)[0]) + 5
        add(n, f, K, [0], [n - 1])
        add(n, f, K, [0, 0, 0], [f + 1, n // 2, n - 2])
        # key 0 from a clamped chain
        K = int(np.flatnonzero(clamp_steps(n) == f)[-1])
        add(n, f, K, [0], [n // 3])
        # key 65535: node 0 measured on it (a measured duplicate), and a fill key of 65535
        add(n, 0, KEYS - 1, on_key=KEYS - 1, count=1)
        add(n, 0, KEYS - 1, on_key=KEYS - 1, count=3)
        fk_all = fill_keys(key_deg(np.arange(KEYS))[:, None], np.arange(1, min(n, 64))[None, :], step_of(n))
        hit = np.argwhere(fk_all == KEYS - 1)
        if len(hit):
            K, i = int(hit[0, 0]), int(hit[0, 1]) + 1
            add(n, 0, K, [i], [n - 1])
            add(n, 0, K, [i], [i + 1] if i + 1 < n else [n - 1])
    for n in SHARED_NS + (1024, 2047):
        e = exact360(n)
        if len(e):  # key 0 from the 360.0f fill: a twin behind and one ahead of the fill node
            K, i = (int(v) for v in e[len(e) // 2])
            add(n, 0, K, [i], [n - 1 if i < n - 1 else 1])
            add(n, 0, K, [i, i], [max(1, i - 1) if i > 1 else n - 1, n - 1 if i < n - 1 else 1])
            add(n, 0, K, on_key=0, count=2)
    # Mode A measured duplicates together with fill duplicates: two measured nodes on one key plus fill twins
    for n in (360, 3200, 8192):
        for d in (1, 5, 15):
            K = int(rng.integers(0, KEYS))
            c = Cases([n], [0], [K])
            fk = final_keys_of(c, 0)
            pos = rng.permutation(np.arange(1, n))[: 2 * d + 1]
            ex = [(int(pos[2 * d]), K)] + [(int(j), int(fk[i])) for i, j in zip(pos[:d], pos[d:2 * d])]
            scans.append((n, 0, K, ex))
    ex = [(s, j, k) for s, (_, _, _, e) in enumerate(scans) for j, k in e]
    return Cases([x[0] for x in scans], [x[1] for x in scans], [x[2] for x in scans], ex)


def extreme_cases():
    """n = 1 (measured and not), f = n - 1, all-unmeasured scans (OPERATION_FAIL, buffer untouched)"""
    return Cases.cat([Cases([1, 1, 1, 2, 2, 5, 360, 8192], [0, 0, -1, 1, -1, 4, 359, -1],
                            [0, 65535, 0, 65535, 0, 12345, 0, 0]),
                      Cases([360, 3200, 8191, 8192], [359, 3199, 8190, 8191], [65535, 65535, 65535, 65535])])


# ---- 3. the checker (torch: CPU and device) ------------------------------------------------------------------------
def t_key_deg(k):
    return k.to(torch.float32) * 90.0 / 16384.0  # exact: k * 90 < 2^23, then a power of two


def t_deg_key(v):
    # v * 16384 is exact; the division by 90 goes through a tensor (tensor / python_scalar multiplies by 1/90)
    return ((v * 16384.0) / torch.full_like(v, 90.0)).to(torch.int64) & 0xFFFF


def t_final_keys(words, counts):
    """(final key of every node [S, W], live [S, W], any measured [S]) by the restatement in torch"""
    dev = words.device
    S, W = words.shape
    col = torch.arange(W, device=dev)[None, :]
    live = col < counts[:, None]
    meas = live & (((words >> 16) & 0xFFFFFFFF) != 0)
    anym = meas.any(1)
    f = torch.where(anym, meas.to(torch.int8).argmax(1), torch.zeros_like(counts))
    K = words.gather(1, f[:, None])[:, 0] & 0xFFFF
    nf = counts.clamp(min=1).to(torch.float32)
    step = torch.full_like(nf, 360.0) / nf
    k = K.clone()
    top = int(f.max()) if S else 0
    for t in range(top):
        act = (f > t) & (k != 0)
        if t % 256 == 0 and not bool(act.any()):
            break
        k = torch.where(act, t_deg_key((t_key_deg(k) - step).clamp(min=0.0)), k)
    front = t_key_deg(k)
    a = front[:, None] + col.to(torch.float32) * step[:, None]
    fill = t_deg_key(torch.where(a > 360.0, a - 360.0, a))
    final = torch.where(meas, words & 0xFFFF, torch.where(col == 0, k[:, None], fill))
    return final, live, anym


def expected(words, counts):
    """(status [S], ascended words [S, W] with SENTINEL behind each count, final keys, live, order) in torch"""
    final, live, anym = t_final_keys(words, counts)
    W = words.shape[1]
    col = torch.arange(W, device=words.device)[None, :]
    big = torch.iinfo(torch.int64).max
    srt = torch.where(live, final * _SPREAD + col, torch.full_like(final, big)).sort(1).values
    idx = torch.where(srt == big, torch.zeros_like(srt), srt & (_SPREAD - 1))
    out = ((words & ~0xFFFF) | final).gather(1, idx)
    out = torch.where(anym[:, None], out, words)
    out = torch.where(live, out, torch.full_like(out, SENTINEL))
    status = torch.where(anym, torch.full_like(counts, OK), torch.full_like(counts, FAIL))
    return status, out, final, live, srt


def shared_counts(words, counts):
    """(D, DM) per scan: nodes beyond the first of their final key, measured nodes beyond the first of their key"""
    _, _, final, live, srt = expected(words, counts)
    sk = srt >> 17
    d = live.sum(1) - (((sk[:, 1:] != sk[:, :-1]) & live[:, 1:]).sum(1) + live[:, 0].to(torch.int64))
    meas = live & (((words >> 16) & 0xFFFFFFFF) != 0)
    mk = torch.where(meas, words & 0xFFFF, torch.full_like(words, KEYS)).sort(1).values
    m = meas.sum(1)
    dm = m - (((mk[:, 1:] != mk[:, :-1]) & (mk[:, 1:] < KEYS)).sum(1) + (mk[:, 0] < KEYS).to(torch.int64))
    return d, dm


def _t(a, dev=None):
    if isinstance(a, torch.Tensor):
        return a.to(torch.int64)
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.int64))).to(dev or "cpu")


def first_ascend_mismatch(got, status, words, counts):
    """(scan, slot or -1 for the status, got, want) of the first difference between a kernel's ascended buffers
    (got [S, W] int64 words, the slots behind each count included: they must still hold SENTINEL) and status, and the
    restatement; None if none.  numpy arrays or torch tensors (on any device)."""
    got, words = _t(got), _t(words)
    dev = words.device
    status, counts = _t(status, dev).to(dev) & 0xFFFFFFFF, _t(counts, dev).to(dev)  # (a u32 read through int32)
    got = got.to(dev)
    want_st, want, *_ = expected(words, counts)
    bad = (status != want_st).nonzero()
    if bad.numel():
        s = int(bad[0])
        return s, -1, int(status[s]), int(want_st[s])
    ok = got == want
    if bool(ok.all()):
        return None
    s, j = (int(v) for v in (~ok).nonzero()[0])
    return s, j, int(got[s, j]), int(want[s, j])


def describe(where, words, counts):
    s, j, g, w = where
    n = int(counts[s])
    if j < 0:
        return f"scan {s} (n {n}): status {g:#x}, want {w:#x}"
    if j >= n:
        return f"scan {s} (n {n}): slot {j} behind the count was written ({g:#018x})"
    return (f"scan {s} (n {n}): slot {j} holds {g:#018x} (key {g & 0xFFFF}), want {w:#018x} (key {w & 0xFFFF})")


# ---- the CPU tests ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref(oracle):
    return Reference(oracle)


def test_exact_360_fills_are_counted_as_the_float_arithmetic_gives_them():
    """The fills that land on exactly 360.0f, over every front key and every i: a few at most n, every i at the
    powers of two (i * step and 360 - deg(K) are then both exact)"""
    assert {n: len(exact360(n)) for n in (360, 3200, 8191, 4096, 8192)} == {360: 7, 3200: 127, 8191: 54, 4096: 4095,
                                                                            8192: 8191}
    for n in (360, 3200, 4096, 8191):  # against a brute force over every (K, i)
        a = key_deg(np.arange(KEYS))[:, None] + np.arange(1, n)[None, :].astype(F32) * step_of(n)
        K, i = np.nonzero(a == F32(360.0))
        assert (np.stack([K, i + 1], 1) == exact360(n)).all(), n
    have = [n for n in range(1, 8193) if len(exact360(n))]
    assert len(have) > 1000 and all(len(exact360(n)) for n in SHARED_NS if n in (360, 720, 1000, 3200, 4096, 8191, 8192))


def test_restatement_fill_reaches_key_zero_at_360_and_the_wrap():
    for n in (360, 3200, 4096, 8191, 8192):
        K, i = exact360(n)[0]
        st, out = ascend_words(fill_cases(n, [K]).words(n), [n])
        assert st[0] == OK and (out[0] & 0xFFFF)[0] == 0, n  # the 360.0f node sorts first with key 0
        assert fill_keys(key_deg(K), i, step_of(n)) == 0
        assert fill_keys(key_deg(K), i, step_of(n), ge=True) == 0  # ... as does the faulty >= (0.0f)
        # the wrap: some node past 360 comes back near 0, the keys before it stay above the front key
        fk = fill_keys(key_deg(K), np.arange(1, n), step_of(n))
        assert (fk < K).any() and (fk > K).any()


@pytest.mark.parametrize("n", CHAIN_NS)
def test_head_chain_map_and_clamp_edges(n):
    """g_n is monotone and strictly below k for k > 0; the clamp edges clamp at f - 1, f, f + 1 steps; iterating the
    map gives what the walk gives, for every f of the chain families"""
    g = chain_map(n)
    k = np.arange(KEYS)
    assert g[0] == 0 and (g[1:] < k[1:]).all() and (np.diff(g) >= 0).all()
    c = clamp_steps(n)
    assert (np.diff(c) >= 0).all()
    reach = set()
    for f in sorted({1, 2, n // 2, n - 1} | set(range(1, min(n, 64)))):
        e = clamp_edge_keys(n, f)
        if not len(e):
            continue
        reach |= {int(c[x]) - f for x in e}
        assert (chain_power(n, f)[e] == head_keys(e, np.full(len(e), f), step_of(n))).all()
        assert (chain_power(n, f)[e[c[e] <= f]] == 0).all() and (chain_power(n, f)[e[c[e] > f]] != 0).all()
    assert reach >= {-1, 0, 1} or n < 4  # short of the clamp, exactly at f and one step later
    K = np.arange(0, KEYS, 97)
    for f in (1, 2, n // 2, n - 1):
        assert (chain_power(n, f)[K] == head_keys(K, np.full(len(K), f), step_of(n))).all()


def test_case_builders_reach_the_edges():
    for n in (360, 3200, 8192):
        cb = chain_cases(n)
        assert set(cb.f.tolist()) == set(range(n))
        c = clamp_steps(n)
        exact = cb.f == c[cb.K]
        assert exact.sum() >= n // 2 and (c[cb.K] == cb.f + 1).any() and ((c[cb.K] == cb.f - 1) & (cb.f > 0)).any()
    ex = extreme_cases()
    st, out = ascend_words(ex.words(8192), ex.n)
    assert (st == FAIL).sum() == 3 and set(ex.n.tolist()) >= {1, 2} and (ex.f == ex.n - 1).sum() >= 5
    w = ex.words(8192)
    bad = st == FAIL
    assert (out[bad][:, :1] == w[bad][:, :1]).all()  # untouched
    # shared final keys: D = 0..17, key 0 (360.0f fill and clamped chain), key 65535, four nodes on one key, the twin
    # before and after the node it shares a key with
    sc = shared_key_cases()
    W = int(sc.n.max())
    words = sc.words(W)
    d, dm = (v.numpy() for v in shared_counts(torch.from_numpy(words), torch.from_numpy(sc.n)))
    assert set(range(MAX_DUP + 1)) <= set(d.tolist())
    assert (dm > 0).any() and ((dm > 0) & (d > dm)).any()  # measured duplicates together with fill duplicates
    final, live, _ = t_final_keys(torch.from_numpy(words), torch.from_numpy(sc.n))
    final = torch.where(live, final, torch.full_like(final, -1)).numpy()
    shared = set()
    most = 0
    before_after = set()
    for s in range(len(sc)):
        fk = final[s][: sc.n[s]]
        keys, cnt = np.unique(fk, return_counts=True)
        most = max(most, cnt.max())
        meas = ((words[s, : sc.n[s]] >> 16) & 0xFFFFFFFF) != 0
        for k in keys[cnt > 1]:
            pos = np.flatnonzero(fk == k)
            shared.add(int(k))
            before_after.add((bool(meas[pos[0]]), bool(meas[pos[-1]])))
            if k == 0 and not meas[pos].all():
                shared.add("0 from " + ("chain" if pos[0] == 0 and sc.f[s] > 0 else "fill"))
    assert {0, KEYS - 1, "0 from chain", "0 from fill"} <= shared and most >= 4
    assert {(True, False), (False, True)} <= before_after


def _sample_scans():
    """A sample of every family, as (words, counts) of one width"""
    rng = np.random.default_rng(5)
    parts = [fill_cases(n, rng.choice(KEYS, 3, replace=False)) for n in SHARED_NS + WIDE_NS[:1]]
    parts += [fill_cases(n, exact360_keys(n)[:2]) for n in SHARED_NS if len(exact360(n))]
    for n in (5, 64, 360, 3200):
        cb = chain_cases(n)
        parts.append(cb.take(rng.choice(len(cb), 6, replace=False)))
    parts.append(chain_every_key_cases(360, 4099))
    parts.append(extreme_cases())
    sc = shared_key_cases()
    parts.append(sc.take(np.arange(0, len(sc), 3)))
    c = Cases.cat(parts)
    return c.words(int(c.n.max())), c.n


@pytest.fixture(scope="module")
def sample():
    return _sample_scans()


def _by_key(out):
    keys, cnt = np.unique(out["angle_z_q14"], return_counts=True)
    uniq = np.isin(out["angle_z_q14"], keys[cnt == 1])
    return np.ascontiguousarray(out["angle_z_q14"]), np.sort(out.view(np.uint64)), out.view(np.uint64)[uniq]


def test_restatement_equals_the_reference_and_the_oracle(ref, sample):
    """Every sample scan: the reference's ascendScanData (bit for bit where no two nodes share a final key; the key
    sequence and per-key multiset otherwise -- its std::sort is not stable) and oracle/scan_oracle.cpp with the stable
    rule (bit for bit)"""
    words, counts = sample
    st, out = ascend_words(words, counts)
    ties = 0
    for s in range(len(counts)):
        n = int(counts[s])
        nodes = np.ascontiguousarray(words[s, :n]).view(ref.NODE_DTYPE)
        mine = out[s, :n].view(ref.NODE_DTYPE)
        rc_o, out_o = ref.ascend(nodes, stable=True)
        assert rc_o == st[s] and same(out_o, mine), s
        if len(np.unique(mine["angle_z_q14"])) == n or st[s] == FAIL:
            rc_r, out_r = ref.ref_ascend(nodes)
            assert rc_r == st[s] and same(mine, out_r), s
        else:
            ties += 1
            r_keys, r_all, r_uniq = ref.call("ref_ascend", nodes, post=lambda r: _by_key(r[1]))
            m_keys, m_all, m_uniq = _by_key(mine)
            assert same(m_keys, r_keys) and same(m_all, r_all) and same(m_uniq, r_uniq), s
    assert ties >= 40


def test_torch_restatement_equals_numpy(sample):
    words, counts = sample
    st, out = ascend_words(words, counts)
    t_st, t_out, *_ = expected(torch.from_numpy(words), torch.from_numpy(counts))
    assert (t_st.numpy() == st).all() and (t_out.numpy() == out).all()
    v = torch.from_numpy(key_deg(np.arange(KEYS)) + F32(0.7))
    assert (t_deg_key(v).numpy() == deg_key(v.numpy())).all()
    a = np.arange(0, 721 * 64, dtype=F32) / F32(64)  # every angle on a 1/64 grid up to 720: many exact quotients
    assert (t_deg_key(torch.from_numpy(a)).numpy() == deg_key(a)).all()


# ---- 4. planted faults -----------------------------------------------------------------------------------------------
FAULTS = {
    "fill rounded once (FMA)": dict(fma=True),
    "head chain quantised once": dict(chain="once"),
    "head chain one step short": dict(chain_short=1),
    "step = 360 / (n - 1)": dict(step_n1=True),
    "node 0 given the fill formula": dict(chain="fill"),
    "shared keys in reverse buffer order": dict(reverse_ties=True),
}


def fault_scans():
    """What the faults are run on: the sample, the exact-360 scans of every swept n, every key at the small n and
    f = 1, and every 61st key at n = 1000, 3200, 8191"""
    rng = np.random.default_rng(3)
    parts = [fill_cases(n, spread(exact360_keys(n), 64)) for n in SHARED_NS if len(exact360(n))]
    parts += [fill_cases(n, np.arange(KEYS)) for n in (2, 3, 12)]
    parts += [fill_cases(n, np.arange(0, KEYS, 61)) for n in (1000, 3200, 8191)]
    parts += [chain_every_key_cases(12, 3)]
    for n in (12, 64, 360):
        cb = chain_cases(n)
        parts.append(cb.take(rng.choice(len(cb), min(len(cb), 200), replace=False)))
    parts.append(shared_key_cases())
    return parts


def model_mismatch(**fault):
    for c in fault_scans():
        words = c.words(int(c.n.max()))
        st, out = ascend_words(words, c.n, **fault)
        if first_ascend_mismatch(out, st, words, c.n) is not None:
            return True
    return False


def test_checker_passes_the_unmutated_model(sample):
    words, counts = sample
    st, out = ascend_words(words, counts)
    assert first_ascend_mismatch(out, st, words, counts) is None
    assert not model_mismatch()
    bad = out.copy()
    s = int(np.flatnonzero(counts < words.shape[1])[0])
    bad[s, counts[s]] = 0
    assert first_ascend_mismatch(bad, st, words, counts)[:2] == (s, counts[s])  # a slot written behind n


@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_rejects_a_faulty_model(fault):
    assert model_mismatch(**FAULTS[fault]), f"the sweep cannot see the fault: {fault}"


def test_wrap_at_or_above_360_stores_the_same_key():
    """ascend_fill_key wraps when a > 360.0f; a >= 360.0f would subtract at exactly 360.0f too, giving 0.0f and key 0
    -- the key (u32)65536 stored in a u16 gives as well.  Every exact-360 fill of the sweeps ascends the same way
    under both tests, so that variant is no fault and no sweep can reject it."""
    for n in sorted(set(SHARED_NS) | set(WIDE_NS) | {1000, 2047}):
        K, i = exact360(n).T
        if not len(K):
            continue
        assert (fill_keys(key_deg(K), i, step_of(n)) == 0).all() and (fill_keys(key_deg(K), i, step_of(n), ge=True) == 0).all()
        c = fill_cases(n, np.unique(K)[:64])
        words = c.words(n)
        assert all((a == b).all() for a, b in zip(ascend_words(words, c.n), ascend_words(words, c.n, ge=True)))


def test_wrap_after_quantising_stores_the_same_key():
    """Quantising a fill angle a in (360, 720) and letting the u16 store drop 65536 gives the key of a - 360 for every
    float a there: a is a multiple of 2^-15, so a * 16384 / 90 lies at least 1/180 from the next integer, more than
    half an ulp of the quotient (at most 2^-7).  That variant is no fault either."""
    a = np.arange(np.array(360.0, F32).view(np.int32) + 1, np.array(720.0, F32).view(np.int32), dtype=np.int32).view(F32)
    assert len(a) > 5_000_000
    assert (deg_key(a) == deg_key(a - F32(360.0))).all()
    c = fill_cases(1000, np.arange(0, KEYS, 5))
    words = c.words(1000)
    assert all((x == y).all() for x, y in zip(ascend_words(words, c.n), ascend_words(words, c.n, wrap_after=True)))
