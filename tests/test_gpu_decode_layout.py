"""The wire decoders across their whole stream layout, against the oracle bit for bit.

The other decoder tests lay every stream out 16-byte aligned, write the nodes to a fresh (16-byte aligned) torch
allocation and decode at most 64 streams, so that every CTA decodes one aligned stream.  The entry points accept far
more than that, and other code serves it:

  * stage() in decode_capsule_kernel copies a tile with 16-byte cp.async, 4-byte cp.async or byte loads, chosen by the
    stream base's alignment; the HQ kernel uses 16-byte copies or byte loads (test_alignment_sweep);
  * express, dense and ultra-dense store node pairs as one 16-byte word only when the output is 16-byte aligned, and
    as two 8-byte words otherwise (test_alignment_sweep, node_offset = 8);
  * every decoder and the framer loop over streams when there are more than their grid (num_sms x 4 or 8) and reset
    their per-stream state in between (test_more_streams_than_ctas);
  * the dense entry points list each stream's scan-start nodes through an unordered atomicAdd
    (test_dense_scan_start_list);
  * the timestamp and CDR launchers split a batch into slabs of 65535 streams (test_past_65535_*);
  * sample_duration_us at the ends of its range (test_sample_duration_bounds).

The case builders are checked without a GPU (test_sweep_reaches_every_staging_and_store_branch)."""
import functools

import numpy as np
import pytest

from oracle import cdr_oracle as cdr
from test_capsule_oracle_vs_ref import make_capsules
from test_decode_oracle_vs_ref import make_stream
from test_framing_vs_ref import damaged_stream
from test_timestamps_vs_ref import rx_times

gpu = pytest.mark.gpu

CB = {0x82: 84, 0x83: 781, 0x84: 132, 0x85: 84, 0x86: 170}  # bytes per capsule
PER = {0x82: 32, 0x83: 96, 0x84: 96, 0x85: 40, 0x86: 64}    # nodes per capsule
DT = {0x82: 256, 0x83: 32, 0x84: 256, 0x85: 256, 0x86: 128}  # capsules per tile of the format's kernel
FORMATS = tuple(CB)
FRAMED = (0x82, 0x84, 0x85, 0x86)  # formats the byte-level framer serves
# per format: a stride that keeps every stream 16-byte aligned, and an odd one whose streams start in several
# classes mod 16; both hold the longest ragged stream (2 * DT + 3 capsules)
STRIDES = {0x82: (516, 517), 0x83: (80, 69), 0x84: (516, 517), 0x85: (516, 517), 0x86: (264, 261)}
BASE_OFFSETS = (0, 2, 4, 8, 12)
NODE_OFFSETS = (0, 8)
NODE_FILL = 0xCD
WORD_FILL = 0xDEADBEEF
WORD_FILL_I32 = int(np.array(WORD_FILL, np.uint32).view(np.int32))
SLAB = 65535  # streams per grid.y slab of the timestamp and CDR launchers


def ragged_counts(ans):
    d = DT[ans]
    return (0, 1, d - 1, d, d + 1, 2 * d + 3)


def sweep_cases():
    """(ans, entry, base_offset, stride_capsules, node_offset).  entry "capsules": rpl_decode_capsules_batch_dev (two
    state words per stream); "dense": rpl_decode_dense_batch_dev (one).  Dense streams must start 4-byte aligned."""
    cases = []
    for ans in FORMATS:
        for entry in (("capsules", "dense") if ans == 0x85 else ("capsules",)):
            for base in BASE_OFFSETS:
                if ans == 0x85 and base % 4:
                    continue
                for stride in STRIDES[ans]:
                    for node_offset in NODE_OFFSETS:
                        cases.append((ans, entry, base, stride, node_offset))
    return cases


def stream_bases(ans, base_offset, stride, n_streams):
    """Byte offset of each stream from a 16-byte aligned allocation.  Every tile of a stream starts in the same class
    mod 16 as the stream (DT * CB is a multiple of 16 for every format)."""
    return [base_offset + s * stride * CB[ans] for s in range(n_streams)]


# ---- batches on the device ------------------------------------------------------------------------------------------
def lay_out(streams, cb, per, stride, base_offset, node_offset, state_words, states):
    """Device buffers of one batch.  Stream s starts s * stride * cb bytes after data_ptr() + base_offset, and every
    byte outside the live capsules is 0xEE.  nodes_out starts node_offset bytes into its allocation, which is NODE_FILL
    throughout; the status, offset, count and state-out words are WORD_FILL."""
    import torch

    dev = torch.device("cuda")
    n = len(streams)
    host = np.full(base_offset + n * stride * cb + 16, 0xEE, np.uint8)
    for s, c in enumerate(streams):
        assert len(c) <= stride
        o = base_offset + s * stride * cb
        host[o: o + c.size] = c.reshape(-1)
    buf = torch.from_numpy(host).to(dev)
    nodes = torch.full((node_offset + n * stride * per * 8 + 16,), NODE_FILL, dtype=torch.uint8, device=dev)
    assert buf.data_ptr() % 16 == 0 and nodes.data_ptr() % 16 == 0

    def words(k):
        return torch.full((k,), WORD_FILL_I32, dtype=torch.int32, device=dev)

    st = np.array([tuple(x)[:state_words] for x in states], np.uint32).reshape(-1)
    L = dict(n=n, cb=cb, per=per, stride=stride, node_offset=node_offset, state_words=state_words, buf=buf,
             nodes_t=nodes, caps=buf.data_ptr() + base_offset, nodes=nodes.data_ptr() + node_offset,
             counts_h=np.array([len(c) for c in streams], np.uint32), ncount=words(n), status=words(n * stride),
             offs=words(n * stride), state_in=torch.from_numpy(st.view(np.int32)).to(dev),
             state_out=words(n * state_words))
    L["counts"] = torch.from_numpy(L["counts_h"].view(np.int32)).to(dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    return L


def decode(ctx, ans, entry, L, sample_us=31, **starts):
    if entry == "dense":
        ctx.decode_dense_batch_dev(L["caps"], L["counts"].data_ptr(), L["n"], L["stride"], sample_us, L["nodes"],
                                   L["ncount"].data_ptr(), sync_state_in=L["state_in"].data_ptr(),
                                   capsule_status=L["status"].data_ptr(), capsule_node_offset=L["offs"].data_ptr(),
                                   sync_state_out=L["state_out"].data_ptr(), **starts)
    else:
        ctx.decode_capsules_batch_dev(ans, L["caps"], L["counts"].data_ptr(), L["n"], L["stride"], sample_us,
                                      L["nodes"], L["ncount"].data_ptr(), state_in=L["state_in"].data_ptr(),
                                      capsule_status=L["status"].data_ptr(), capsule_node_offset=L["offs"].data_ptr(),
                                      state_out=L["state_out"].data_ptr())
    ctx.synchronize()


def expected_state(ans, est, state_words):
    """The state words the decoder leaves: the scan-start flag (dense, ultra-dense) and the last distance
    (ultra-dense); 0 where the format keeps no such state.  One word in the dense entry points' layout."""
    if state_words == 1:
        return (est[0],)
    return {0x85: (est[0], 0), 0x86: tuple(est)}.get(ans, (0, 0))


def check_batch(O, ans, L, expected, only=None):
    """Every stream (or those in `only`) against the oracle's (nodes, status, offsets, state) for its own capsules and
    state; the fill must be untouched past each stream's node and capsule counts."""
    import torch

    torch.cuda.synchronize()
    n, stride, per, sw = L["n"], L["stride"], L["per"], L["state_words"]
    raw = L["nodes_t"].cpu().numpy()
    no = L["node_offset"]
    body = raw[no: no + n * stride * per * 8]
    assert (raw[:no] == NODE_FILL).all() and (raw[no + body.size:] == NODE_FILL).all()
    hn = body.view(np.uint64).reshape(n, stride * per)
    fill64 = np.uint64(int.from_bytes(bytes([NODE_FILL] * 8), "little"))
    hc = L["ncount"].cpu().numpy().view(np.uint32)
    hs = L["status"].cpu().numpy().view(np.uint32).reshape(n, stride)
    ho = L["offs"].cpu().numpy().view(np.uint32).reshape(n, stride)
    hst = L["state_out"].cpu().numpy().view(np.uint32).reshape(n, sw)
    for s in (range(n) if only is None else only):
        en, es, eo, est = expected[s]
        k = int(L["counts_h"][s])
        m = len(en)
        where = (hex(ans), s, k)
        assert hc[s] == m, where + (int(hc[s]), m)
        bad = np.flatnonzero(hn[s, :m] != en.view(np.uint64))
        assert bad.size == 0, where + (bad[:8],)
        assert (hn[s, m:] == fill64).all(), where  # nothing written past the stream's nodes
        assert (hs[s, :k] == es).all() and (hs[s, k:] == WORD_FILL).all(), where
        assert (ho[s, :k] == eo).all() and (ho[s, k:] == WORD_FILL).all(), where
        assert tuple(int(x) for x in hst[s]) == expected_state(ans, est, sw), where


# ---- the alignment sweep --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def sweep_streams(O, ans):
    """Ragged streams around the format's tile, each with its entering state, and the oracle's decode of each.
    Scan-start capsules, checksum errors, errors across the first tile boundary with a broken marker on the second
    tile's first capsule; ultra-dense streams of near-range samples, so that the smoothing chain crosses tiles."""
    d = DT[ans]
    rng = np.random.default_rng(ans)
    streams = []
    for i, n in enumerate(ragged_counts(ans)):
        if ans == 0x85:
            caps = make_stream(O, n, 40.0 + i, seed=900 + i, sync_every=60 + i)
        else:
            caps = make_capsules(O, ans, n, 40.0 + i, seed=900 + i, sync_every=None if ans == 0x83 else 60 + i,
                                 near=ans == 0x86)
        if n > 2:
            caps[rng.choice(n, max(1, n // 40), replace=False), 20] ^= 0x08
        if n > d:
            caps[d - 2: d + 2, 30] ^= 0xFF
            caps[d, 0] = 0x00 if ans == 0x83 else 0x30
        streams.append(caps)
    states = [(s & 1, (0, 800, 3000)[s % 3]) for s in range(len(streams))]
    expected = [O.decode_capsules(ans, c, 31, st) for c, st in zip(streams, states)]
    return streams, states, expected


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 8192, 64)
    yield c
    c.close()


@gpu
@pytest.mark.parametrize("ans, entry, base_offset, stride, node_offset",
                         [pytest.param(*c, id="%#x-%s-base%d-stride%d-nodes%d" % c) for c in sweep_cases()])
def test_alignment_sweep(oracle, ctx, ans, entry, base_offset, stride, node_offset):
    streams, states, expected = sweep_streams(oracle, ans)
    L = lay_out(streams, CB[ans], PER[ans], stride, base_offset, node_offset, 1 if entry == "dense" else 2, states)
    decode(ctx, ans, entry, L)
    check_batch(oracle, ans, L, expected)


@gpu
@pytest.mark.parametrize("entry", ["capsules", "dense"])
def test_dense_streams_must_be_4_byte_aligned(R, oracle, ctx, entry):
    streams, states, _ = sweep_streams(oracle, 0x85)
    L = lay_out(streams, 84, 40, 516, 2, 0, 1 if entry == "dense" else 2, states)
    with pytest.raises(R.RplError):
        decode(ctx, 0x85, entry, L)
    assert (L["ncount"].cpu().numpy() == WORD_FILL_I32).all()  # rejected before anything ran


def test_sweep_reaches_every_staging_and_store_branch():
    """Which branch of the staging and of the node stores each sweep case reaches, from its stream bases (mod 16) and
    its nodes_out alignment.  Fails naming the branch a narrower sweep would leave untested."""
    reached = {}
    for ans, entry, base, stride, node_offset in sweep_cases():
        got = reached.setdefault((ans, entry), set())
        counts = ragged_counts(ans)
        assert max(counts) <= stride and DT[ans] + 1 in counts and 2 * DT[ans] + 3 in counts
        for b in stream_bases(ans, base, stride, len(counts)):
            if b % 16 == 0:
                got.add("16-byte staging")
            elif b % 4 == 0:
                got.add("4-byte staging" if ans != 0x83 else "byte staging")
            else:
                assert ans != 0x85, "dense streams are rejected unless 4-byte aligned"
                got.add("byte staging")
                if b % 2 == 0:
                    got.add("2-byte aligned base")
        got.add("16-byte node stores" if node_offset % 16 == 0 else "8-byte node stores")
    want = {
        (0x82, "capsules"): {"16-byte staging", "4-byte staging", "byte staging", "2-byte aligned base"},
        (0x84, "capsules"): {"16-byte staging", "4-byte staging", "byte staging", "2-byte aligned base"},
        (0x86, "capsules"): {"16-byte staging", "4-byte staging", "byte staging", "2-byte aligned base"},
        (0x83, "capsules"): {"16-byte staging", "byte staging", "2-byte aligned base"},
        (0x85, "capsules"): {"16-byte staging", "4-byte staging"},
        (0x85, "dense"): {"16-byte staging", "4-byte staging"},
    }
    for key, branches in want.items():
        branches = branches | {"16-byte node stores", "8-byte node stores"}
        missing = branches - reached.get(key, set())
        assert not missing, f"{key[0]:#x} via the {key[1]} entry point no longer reaches: {sorted(missing)}"


# ---- more streams than CTAs -----------------------------------------------------------------------------------------
def num_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def many_capsule_streams(O, ans, n_streams, grid):
    """Short streams (3..40 capsules, some empty) in which a per-stream state that leaked from stream s - grid (the
    previous stream of the same CTA) would change stream s: every stream starts on a valid capsule that is not a scan
    start and ends on a valid one, and each stream's entering state differs from the state stream s - grid leaves."""
    rng = np.random.default_rng(7000 + ans)
    counts = rng.integers(3, 41, n_streams)
    counts[rng.random(n_streams) < 0.08] = 0
    streams, states, expected = [], [], []
    for s in range(n_streams):
        n = int(counts[s])
        # one capsule more, and the first (a scan start when sync_every is set) dropped
        if ans == 0x85:
            caps = make_stream(O, n + 1, 30.0, seed=s, sync_every=12 + s % 17)[1:]
        else:
            caps = make_capsules(O, ans, n + 1, 30.0, seed=s, sync_every=None if ans == 0x83 else 12 + s % 17,
                                 near=ans == 0x86)[1:]
        if n >= 3 and s % 5 == 0:
            caps[int(rng.integers(1, n - 1)), 20] ^= 0x08  # a checksum error inside the stream
        if s < grid:
            st = (s & 1, 0 if s % 4 < 2 else 2000)
        else:
            prev = expected[s - grid][3]
            st = (1 - (prev[0] & 1), prev[1] + 4)
        streams.append(np.ascontiguousarray(caps))
        states.append(st)
        expected.append(O.decode_capsules(ans, caps, 31, st))
    return streams, states, expected


@gpu
@pytest.mark.parametrize("ans, entry", [pytest.param(a, e, id=f"{a:#x}-{e}") for a, e in
                                        [(a, "capsules") for a in FORMATS] + [(0x85, "dense")]])
def test_more_streams_than_ctas_capsules(oracle, ctx, ans, entry):
    grid = num_sms() * (4 if ans == 0x85 else 8)  # decode_capsules_launch
    n_streams = 3 * num_sms() * 8 + 5
    assert n_streams > 3 * grid
    streams, states, expected = many_capsule_streams(oracle, ans, n_streams, grid)
    if entry == "dense":
        expected = [(en, es, eo, (est[0], 0)) for en, es, eo, est in expected]
    L = lay_out(streams, CB[ans], PER[ans], 40, 0, 0, 1 if entry == "dense" else 2, states)
    decode(ctx, ans, entry, L)
    check_batch(oracle, ans, L, expected)


def standard_records(rng, n):
    rec = np.zeros((n, 5), np.uint8)
    sb = (rng.random(n) < 0.05).astype(np.uint8)
    rec[:, 0] = (rng.integers(0, 64, n).astype(np.uint8) << 2) | ((1 - sb) << 1) | sb
    w = (rng.integers(0, 360 * 64, n).astype(np.uint16) << 1) | 1
    rec[:, 1], rec[:, 2] = w & 0xFF, w >> 8
    rec[:, 3:] = rng.integers(0, 256, (n, 2))
    return rec.reshape(-1)


@gpu
def test_more_streams_than_ctas_standard_nodes(oracle, ctx):
    """0x81 byte streams: the streams of every other pass of a CTA end inside a record, and the stream its CTA takes
    next is clean, so a byte-machine state or 4-byte halo left from the previous stream would misframe it."""
    import torch

    grid = num_sms() * 8
    n_streams = 3 * grid + 5
    rng = np.random.default_rng(81)
    stride = 600
    streams = []
    for s in range(n_streams):
        b = standard_records(rng, int(rng.integers(3, 120)))
        if (s // grid) % 2 == 0:
            b = b[: len(b) - int(rng.integers(1, 5))]  # ends inside a record
        if s % 11 == 0:
            b = b[:0]
        if s % 7 == 3 and len(b) > 20:
            b = b.copy()
            b[int(rng.integers(0, len(b)))] ^= 0xFF
        streams.append(b)
    host = np.full((n_streams, stride), 0xEE, np.uint8)
    for s, b in enumerate(streams):
        host[s, : len(b)] = b
    dev = torch.device("cuda")
    wire = torch.from_numpy(host).to(dev)
    counts = torch.tensor([len(b) for b in streams], dtype=torch.int32, device=dev)
    per = stride // 5
    nodes = torch.full((n_streams, per, 8), NODE_FILL, dtype=torch.uint8, device=dev)
    ncount = torch.full((n_streams,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    fsm = torch.full((n_streams,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    ends = torch.full((n_streams, per), WORD_FILL_I32, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_normal_batch_dev(wire.data_ptr(), counts.data_ptr(), n_streams, stride, nodes.data_ptr(),
                                ncount.data_ptr(), fsm_state_out=fsm.data_ptr(), node_end=ends.data_ptr())
    ctx.synchronize()
    hn = nodes.cpu().numpy().view(np.uint64).reshape(n_streams, per)
    hc, hf = ncount.cpu().numpy(), fsm.cpu().numpy()
    he = ends.cpu().numpy().view(np.uint32)
    fill64 = np.uint64(int.from_bytes(bytes([NODE_FILL] * 8), "little"))
    mid_record = 0
    for s, b in enumerate(streams):
        en, eend, epos = oracle.decode_normal(b)
        m = len(en)
        assert hc[s] == m and hf[s] == epos, (s, int(hc[s]), m, int(hf[s]), epos)
        assert (hn[s, :m] == en.view(np.uint64)).all() and (hn[s, m:] == fill64).all(), s
        assert (he[s, :m] == eend).all() and (he[s, m:] == WORD_FILL).all(), s
        mid_record += epos != 0
    assert mid_record > grid  # the construction did end streams inside a record


@gpu
@pytest.mark.parametrize("ans", [pytest.param(a, id=f"{a:#x}") for a in FRAMED])
def test_more_streams_than_ctas_framer(R, oracle, ctx, ans):
    import torch

    grid = num_sms() * 8
    n_streams = 3 * grid + 5
    cb = CB[ans]
    rng = np.random.default_rng(300 + ans)
    streams = [damaged_stream(oracle, ans, rng, ncap=int(rng.integers(3, 41)), max_edits=2) for _ in range(n_streams)]
    for s in range(0, n_streams, 13):
        streams[s] = streams[s][:0]
    stride_bytes = max(len(b) for b in streams)
    host = np.full((n_streams, stride_bytes), 0xEE, np.uint8)
    for s, b in enumerate(streams):
        host[s, : len(b)] = b
    stride_caps = 2 * (stride_bytes // cb) + 2
    dev = torch.device("cuda")
    raw = torch.from_numpy(host).to(dev)
    counts = torch.tensor([len(b) for b in streams], dtype=torch.int32, device=dev)
    caps = torch.full((n_streams, stride_caps, cb), 0xEE, dtype=torch.uint8, device=dev)
    ccount = torch.full((n_streams,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    left = torch.full((n_streams,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.frame_capsules_dev(ans, raw.data_ptr(), counts.data_ptr(), n_streams, stride_bytes, caps.data_ptr(),
                           stride_caps, ccount.data_ptr(), bytes_left_out=left.data_ptr())
    ctx.synchronize()
    hc, hn, hl = caps.cpu().numpy(), ccount.cpu().numpy(), left.cpu().numpy()
    unfinished = 0
    for s, b in enumerate(streams):
        exp, eleft = oracle.frame_capsules(ans, b)
        assert hn[s] == exp.shape[0] and hl[s] == eleft, (hex(ans), s, int(hn[s]), exp.shape[0], int(hl[s]), eleft)
        assert (hc[s, : hn[s]] == exp).all() and (hc[s, hn[s]:] == 0xEE).all(), (hex(ans), s)
        unfinished += eleft != 0
    assert unfinished > 0


# ---- the dense scan-start list --------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("base_offset", [0, 4])
def test_dense_scan_start_list(oracle, ctx, base_offset):
    """scan_start_counts[s] is the number of nodes with flag bit 0; the list holds their positions (in no order) when it
    fits in starts_stride, and otherwise starts_stride of them, with nothing written past the last stream's slot."""
    import torch

    # (capsules, capsules per revolution): ~1 start per 80 capsules up to ~1 per 9 (each below the jump threshold)
    specs = [(200, 80.0), (0, 80.0), (1, 80.0), (257, 40.0), (300, 9.0), (513, 12.0), (90, 80.0), (256, 9.5), (40, 9.0)]
    streams = [make_stream(oracle, n, cpr, seed=50 + i, sync_every=70 if i % 2 else None) for i, (n, cpr) in
               enumerate(specs)]
    states = [(i % 2, 0) for i in range(len(specs))]
    expected = [oracle.decode_capsules(0x85, c, 31, st) for c, st in zip(streams, states)]
    positions = [np.flatnonzero(en["flag"] & 1).astype(np.uint32) for en, _, _, _ in expected]
    counts = [len(p) for p in positions]
    assert 0 in counts and max(counts) > 20 and 1 <= min(c for c in counts if c) <= 2
    n = len(specs)
    dev = torch.device("cuda")
    for starts_stride in (64, 2):
        L = lay_out(streams, 84, 40, 517, base_offset, 0, 1, states)
        starts = torch.full((n * starts_stride + 32,), WORD_FILL_I32, dtype=torch.int32, device=dev)
        scount = torch.full((n,), WORD_FILL_I32, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        decode(ctx, 0x85, "dense", L, scan_starts=starts.data_ptr(), starts_stride=starts_stride,
               scan_start_counts=scount.data_ptr())
        check_batch(oracle, 0x85, L, [(en, es, eo, (est[0], 0)) for en, es, eo, est in expected])
        hs = starts.cpu().numpy().view(np.uint32)
        hcnt = scount.cpu().numpy().view(np.uint32)
        assert (hs[n * starts_stride:] == WORD_FILL).all()  # nothing past the last slot
        for s in range(n):
            assert hcnt[s] == counts[s], (starts_stride, s, int(hcnt[s]), counts[s])
            slot = hs[s * starts_stride: (s + 1) * starts_stride]
            if counts[s] <= starts_stride:
                assert (np.sort(slot[: counts[s]]) == positions[s]).all(), (starts_stride, s)
                assert (slot[counts[s]:] == WORD_FILL).all(), (starts_stride, s)
            else:  # incomplete: starts_stride distinct scan-start positions
                assert len(set(slot.tolist())) == starts_stride, (starts_stride, s)
                assert np.isin(slot, positions[s]).all(), (starts_stride, s)


# ---- past 65535 streams ---------------------------------------------------------------------------------------------
def sampled(n, seed):
    """The streams either side of the slab boundaries, the last one and 200 at random."""
    fixed = {0, SLAB - 1, SLAB, SLAB + 1, 2 * SLAB - 1, n - 1}
    rng = np.random.default_rng(seed)
    return sorted({i for i in fixed if i < n} | set(rng.choice(n, 200, replace=False).tolist()))


@gpu
def test_past_65535_streams_capsule_timestamps(R, oracle, ctx):
    import torch

    O, ans, per, stride = oracle, 0x82, 32, 3
    n = SLAB + 2 + 1000
    rng = np.random.default_rng(65535)
    host = make_capsules(O, ans, n * stride, 40.0, seed=5, sync_every=97).reshape(n, stride, 84)
    bad = rng.choice(n, 2000, replace=False)
    host[bad, rng.integers(0, stride, bad.size), 20] ^= 0x10
    counts_h = rng.integers(2, stride + 1, n).astype(np.uint32)
    rx_h = rx_times(n * stride, 11).reshape(n, stride)
    timing = (63, 256000, 17, 0)
    dev = torch.device("cuda")
    streams = [host[s, : counts_h[s]] for s in range(n)]
    L = lay_out(streams, 84, per, stride, 0, 0, 2, [(0, 0)] * n)
    rx = torch.from_numpy(rx_h.view(np.int64)).to(dev)
    ts = torch.full((n, stride * per), -1, dtype=torch.int64, device=dev)
    decode(ctx, ans, "capsules", L, sample_us=timing[0])
    torch.cuda.synchronize()
    ctx.node_timestamps_dev(ans, R.Timing(*timing), rx.data_ptr(), L["status"].data_ptr(), L["offs"].data_ptr(),
                            L["counts"].data_ptr(), n, stride, ts.data_ptr())
    ctx.synchronize()
    pick = sampled(n, 1)
    expected = {s: O.decode_capsules(ans, streams[s], timing[0]) for s in pick}
    check_batch(O, ans, L, expected, only=pick)
    hts = ts.cpu().numpy().view(np.uint64)
    for s in pick:
        en, es, eo, _ = expected[s]
        ets = O.node_timestamps(ans, O.timing4(*timing), rx_h[s, : counts_h[s]], es, eo, len(en))
        assert (hts[s, : len(en)] == ets).all(), s
        assert (hts[s, len(en):] == np.uint64(2**64 - 1)).all(), s


@gpu
def test_past_65535_streams_standard_node_timestamps(R, oracle, ctx):
    import torch

    O = oracle
    n = SLAB + 2 + 1000
    rng = np.random.default_rng(81)
    stride, chunk = 20, 8
    stride_chunks = (stride + chunk - 1) // chunk
    host = np.full((n, stride), 0xEE, np.uint8)
    counts_h = np.zeros(n, np.uint32)
    recs = standard_records(rng, n * 4).reshape(n, stride)
    for s in range(n):
        k = 5 * int(rng.integers(2, 5)) - (int(rng.integers(0, 3)) if s % 3 == 0 else 0)
        host[s, :k] = recs[s, :k]
        counts_h[s] = k
    rx_h = rx_times(n * stride_chunks, 12).reshape(n, stride_chunks)
    timing = (476, 115200, 250, 0)
    dev = torch.device("cuda")
    wire = torch.from_numpy(host).to(dev)
    counts = torch.from_numpy(counts_h.view(np.int32)).to(dev)
    nodes = torch.zeros((n, stride // 5, 8), dtype=torch.uint8, device=dev)
    ncount = torch.zeros(n, dtype=torch.int32, device=dev)
    ends = torch.zeros((n, stride // 5), dtype=torch.int32, device=dev)
    rx = torch.from_numpy(rx_h.view(np.int64)).to(dev)
    ts = torch.full((n, stride // 5), -1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_normal_batch_dev(wire.data_ptr(), counts.data_ptr(), n, stride, nodes.data_ptr(), ncount.data_ptr(),
                                node_end=ends.data_ptr())
    ctx.normal_timestamps_dev(R.Timing(*timing), ends.data_ptr(), ncount.data_ptr(), n, stride // 5, chunk,
                              rx.data_ptr(), stride_chunks, ts.data_ptr())
    ctx.synchronize()
    hn = nodes.cpu().numpy().view(np.uint64).reshape(n, stride // 5)
    hc = ncount.cpu().numpy()
    hts = ts.cpu().numpy().view(np.uint64)
    for s in sampled(n, 2):
        en, eend, _ = O.decode_normal(host[s, : counts_h[s]])
        m = len(en)
        assert hc[s] == m and (hn[s, :m] == en.view(np.uint64)).all(), s
        ets = O.normal_timestamps(O.timing4(*timing), eend, chunk, rx_h[s])
        assert (hts[s, :m] == ets).all(), s
        assert (hts[s, m:] == np.uint64(2**64 - 1)).all(), s


@gpu
def test_past_65535_messages_laserscan_cdr(R, ctx):
    import torch

    n, stride, frame_id = 70000, 8, "laser_frame"
    rng = np.random.default_rng(70000)
    ranges_h = (rng.random((n, stride)) * 40).astype(np.float32)
    intens_h = rng.integers(0, 256, (n, stride)).astype(np.float32)
    beams_h = rng.integers(0, stride + 1, n).astype(np.uint32)
    inc_h = rng.random(n).astype(np.float32)
    meta_h = np.zeros(n, R.capi.LASERSCAN_META_DTYPE)
    meta_h["stamp_sec"] = rng.integers(-5, 2_000_000_000, n)
    meta_h["stamp_nanosec"] = rng.integers(0, 1_000_000_000, n)
    for k in ("angle_min", "angle_max", "angle_increment", "time_increment", "scan_time", "range_min", "range_max"):
        meta_h[k] = rng.random(n).astype(np.float32)
    dev = torch.device("cuda")
    ranges, intens = torch.from_numpy(ranges_h).to(dev), torch.from_numpy(intens_h).to(dev)
    beams = torch.from_numpy(beams_h.view(np.int32)).to(dev)
    inc = torch.from_numpy(inc_h).to(dev)
    meta = torch.from_numpy(meta_h.view(np.uint8)).to(dev)
    cdr_stride = (R.lib().rpl_laserscan_cdr_size(len(frame_id), stride) + 15) & ~15
    out = torch.full((n, cdr_stride), 0xEE, dtype=torch.uint8, device=dev)
    sizes = torch.full((n,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.laserscan_cdr_batch_dev(meta.data_ptr(), frame_id, ranges.data_ptr(), intens.data_ptr(), beams.data_ptr(), n,
                                stride, out.data_ptr(), cdr_stride, cdr_sizes=sizes.data_ptr(),
                                angle_increment=inc.data_ptr())
    ctx.synchronize()
    ho, hs = out.cpu().numpy(), sizes.cpu().numpy()
    for s in sampled(n, 3):
        m, b = meta_h[s], int(beams_h[s])
        expect = cdr.laserscan_cdr(int(m["stamp_sec"]), int(m["stamp_nanosec"]), frame_id,
                                   [m["angle_min"], m["angle_max"], inc_h[s], m["time_increment"], m["scan_time"],
                                    m["range_min"], m["range_max"]], ranges_h[s, :b], intens_h[s, :b])
        assert hs[s] == len(expect) and ho[s, : hs[s]].tobytes() == expect, s
        assert (ho[s, hs[s]:] == 0xEE).all(), s


@gpu
def test_past_65535_messages_pointcloud2_cdr(R, ctx):
    import torch

    n, stride, frame_id = 70000, 4, "lidar_3"
    rng = np.random.default_rng(70001)
    xyzi_h = rng.normal(0, 10, (n, stride, 4)).astype(np.float32)
    pcount_h = rng.integers(0, stride + 1, n).astype(np.uint32)
    stamps_h = np.stack([rng.integers(0, 2**31, n), rng.integers(0, 10**9, n)], axis=1).astype(np.uint32)
    dev = torch.device("cuda")
    xyzi = torch.from_numpy(xyzi_h).to(dev)
    pcount = torch.from_numpy(pcount_h.view(np.int32)).to(dev)
    stamps = torch.from_numpy(stamps_h.view(np.int32)).to(dev)
    cdr_stride = (R.lib().rpl_pointcloud2_cdr_size(len(frame_id), stride) + 15) & ~15
    out = torch.full((n, cdr_stride), 0xEE, dtype=torch.uint8, device=dev)
    sizes = torch.full((n,), WORD_FILL_I32, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.pointcloud2_cdr_batch_dev(stamps.data_ptr(), frame_id, xyzi.data_ptr(), pcount.data_ptr(), n, stride,
                                  out.data_ptr(), cdr_stride, cdr_sizes=sizes.data_ptr())
    ctx.synchronize()
    ho, hs = out.cpu().numpy(), sizes.cpu().numpy()
    for s in sampled(n, 4):
        k = int(pcount_h[s])
        expect = cdr.pointcloud2_cdr(int(stamps_h[s, 0]), int(stamps_h[s, 1]), frame_id, xyzi_h[s, :k])
        assert hs[s] == len(expect) and ho[s, : hs[s]].tobytes() == expect, s
        assert (ho[s, hs[s]:] == 0xEE).all(), s


# ---- entry-point boundaries -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("ans, entry", [pytest.param(a, e, id=f"{a:#x}-{e}") for a, e in
                                        [(0x82, "capsules"), (0x85, "capsules"), (0x85, "dense"), (0x86, "capsules")]])
def test_sample_duration_bounds(R, oracle, ctx, ans, entry):
    """1 and 1 000 000 us are decoded (the jump threshold at its largest and smallest); 0 and 1 000 001 are refused."""
    O = oracle
    mk = (lambda n, cpr, seed: make_stream(O, n, cpr, seed=seed, sync_every=50)) if ans == 0x85 else \
         (lambda n, cpr, seed: make_capsules(O, ans, n, cpr, seed=seed, sync_every=50, near=ans == 0x86))
    # ~4.5 degrees per capsule (discarded at 1 us) and ~1 degree per capsule; one revolution per capsule (a step the
    # dense and ultra-dense bound only lets through at 1 000 000 us)
    streams = [mk(300, 80.0, 1), mk(300, 360.0, 2), mk(100, 1.0001, 3)]
    states = [(1, 0), (0, 900), (0, 0)]
    words = 1 if entry == "dense" else 2
    for sample_us in (1, 1_000_000):
        expected = [O.decode_capsules(ans, c, sample_us, st) for c, st in zip(streams, states)]
        L = lay_out(streams, CB[ans], PER[ans], 300, 0, 0, words, states)
        decode(ctx, ans, entry, L, sample_us=sample_us)
        check_batch(O, ans, L, expected)
        if ans in (0x85, 0x86):
            disc = [int(((es & R.capi.CAPSULE_DISCARD) != 0).sum()) for _, es, _, _ in expected]
            assert (disc[0] > 250) if sample_us == 1 else (sum(disc) == 0), (sample_us, disc)
    for sample_us in (0, 1_000_001):
        L = lay_out(streams, CB[ans], PER[ans], 300, 0, 0, words, states)
        with pytest.raises(R.RplError):
            decode(ctx, ans, entry, L, sample_us=sample_us)
