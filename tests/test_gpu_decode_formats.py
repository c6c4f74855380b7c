"""GPU tests of the express / HQ / ultra / ultra-dense capsule decoders and the standard-node byte
machine (SURVEY.md 8(f) rank 1) against the restatement oracle/capsule_oracle.cpp, which
tests/test_capsule_oracle_vs_ref.py pins against the SDK's own unpacker.  Integer work: bit-exact."""
import numpy as np
import pytest

from test_capsule_oracle_vs_ref import make_capsules

pytestmark = pytest.mark.gpu

FORMATS = [0x82, 0x83, 0x84, 0x86]


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 40000, 64)
    yield c
    c.close()


def check(O, ctx, ans, caps, sample_us=31, state=(0, 0)):
    en, es, eo, estate = O.decode_capsules(ans, caps, sample_us, state)
    gn, gs, go, gstate = ctx.decode_capsules(ans, caps, sample_us, state)
    assert len(gn) == len(en)
    bad = np.flatnonzero(gn.view(np.uint64) != en.view(np.uint64))
    assert bad.size == 0, (hex(ans), bad[:8], gn[bad[:4]], en[bad[:4]])
    assert (gs == es).all() and (go == eo).all()
    assert gstate == estate
    return gn, gs


@pytest.mark.parametrize("ans", FORMATS + [0x85])
@pytest.mark.parametrize("n_caps", [1, 2, 3, 127, 128, 129, 255, 256, 257, 700])
def test_clean_streams_across_tile_boundaries(oracle, ctx, ans, n_caps):
    if ans == 0x85:
        from test_decode_oracle_vs_ref import make_stream

        caps = make_stream(oracle, n_caps, 80.0, seed=n_caps)
    else:
        caps = make_capsules(oracle, ans, n_caps, 60.0, seed=n_caps)
    check(oracle, ctx, ans, caps)


@pytest.mark.parametrize("ans", FORMATS)
def test_errors_scan_starts_and_bad_frames(R, oracle, ctx, ans):
    rng = np.random.default_rng(ans)
    caps = make_capsules(oracle, ans, 900, 45.0, seed=100 + ans, sync_every=45)
    caps[rng.choice(900, 50, replace=False), 20] ^= 0x08
    caps[254:259, 30] ^= 0xFF  # errors right on a tile boundary
    caps[511, 0] = 0x30        # broken marker: reported, decoding goes on
    _, st = check(oracle, ctx, ans, caps)
    assert ((st & R.capi.CAPSULE_BAD_FRAME) != 0).sum() == 1
    assert ((st & R.capi.CAPSULE_CHECKSUM_ERR) != 0).sum() >= 50


def test_ultra_dense_smoothing_chain_state_and_threshold(oracle, ctx):
    for seed in range(4):
        caps = make_capsules(oracle, 0x86, 600, 50.0, seed=seed, near=True)
        nodes, _ = check(oracle, ctx, 0x86, caps, state=(seed & 1, 0 if seed < 2 else 1234))
        assert (nodes["dist_mm_q2"] % 8 != 0).mean() > 0.1  # smoothing happened
    # all samples short-range and close together: the chain never breaks inside a capsule
    rng = np.random.default_rng(5)
    caps = make_capsules(oracle, 0x86, 520, 50.0, seed=77, near=True)
    cab = caps[:, 10:].reshape(520, 32, 5)
    cab[:, :, 0] &= 0xFC
    cab[:, :, 2] &= 0xFC
    v = (400 + rng.integers(-1, 2, (520, 64)).cumsum(axis=1) % 3) * 4
    cab[:, :, 0] = (v[:, 0::2] & 0xFC)
    cab[:, :, 1] = (cab[:, :, 1] & 0xF0) | (v[:, 0::2] >> 8)
    cab[:, :, 2] = (v[:, 1::2] & 0xFC)
    cab[:, :, 3] = (cab[:, :, 3] & 0xF0) | (v[:, 1::2] >> 8)
    caps[:, 10:] = cab.reshape(520, 160)
    caps = oracle.seal_capsules(0x86, caps)
    check(oracle, ctx, 0x86, caps)
    for sample_us in (15, 63, 125):
        for cpr in (50.0, 9.0, 4.0):
            check(oracle, ctx, 0x86, make_capsules(oracle, 0x86, 300, cpr, seed=sample_us), sample_us=sample_us)


def test_ultra_special_codes(oracle, ctx):
    from test_capsule_oracle_vs_ref import test_ultra_special_predict_codes_and_zero_majors  # noqa: F401

    rng = np.random.default_rng(4)
    n = 400
    caps = make_capsules(oracle, 0x84, n, 60.0, seed=9)
    words = caps[:, 4:].copy().view("<u4").reshape(n, 32)
    pick = rng.random((n, 32))
    words[pick < 0.15] &= ~np.uint32(0xFFF)
    m = (pick > 0.2) & (pick < 0.3)
    words[m] = (words[m] & ~np.uint32(0x3FF << 12)) | np.uint32(0x200 << 12)
    m = (pick > 0.3) & (pick < 0.4)
    words[m] = (words[m] & ~np.uint32(0x3FF << 22)) | np.uint32(0x1FF << 22)
    m = (pick > 0.5) & (pick < 0.7)
    words[m] = (words[m] & ~np.uint32(0xFFF)) | rng.integers(1, 200, m.sum()).astype(np.uint32)
    caps[:, 4:] = words.view(np.uint8).reshape(n, 128)
    check(oracle, ctx, 0x84, oracle.seal_capsules(0x84, caps))


def test_standard_nodes_byte_machine(oracle, ctx):
    rng = np.random.default_rng(11)
    n = 30000
    rec = np.zeros((n, 5), np.uint8)
    s = (rng.random(n) < 0.01).astype(np.uint8)
    rec[:, 0] = (rng.integers(0, 64, n).astype(np.uint8) << 2) | ((1 - s) << 1) | s
    w = (rng.integers(0, 360 * 64, n).astype(np.uint16) << 1) | 1
    rec[:, 1], rec[:, 2] = w & 0xFF, w >> 8
    rec[:, 3:] = rng.integers(0, 256, (n, 2))
    clean = rec.reshape(-1)
    for stream in (clean, clean[:4], clean[:5], clean[:5119], clean[:5120], clean[:5121], clean[:5125], clean[3:]):
        en, _, _ = oracle.decode_normal(stream)
        gn = ctx.decode_normal(stream)
        assert len(gn) == len(en) and (gn.view(np.uint64) == en.view(np.uint64)).all()
    for seed in range(6):
        r = np.random.default_rng(seed)
        b = clean.copy()
        b[r.choice(len(b), 2000, replace=False)] = r.integers(0, 256, 2000)
        b = np.delete(b, r.choice(len(b), 300, replace=False))
        b = np.insert(b, np.sort(r.choice(len(b), 300, replace=False)), r.integers(0, 256, 300).astype(np.uint8))
        en, _, _ = oracle.decode_normal(b)
        gn = ctx.decode_normal(b)
        assert 0 < len(en) < n and len(gn) == len(en)
        assert (gn.view(np.uint64) == en.view(np.uint64)).all()
    noise = rng.integers(0, 256, 50000, dtype=np.uint8)
    en, _, _ = oracle.decode_normal(noise)
    gn = ctx.decode_normal(noise)
    assert len(gn) == len(en) and (gn.view(np.uint64) == en.view(np.uint64)).all()


@pytest.mark.parametrize("ans", FORMATS + [0x85])
def test_batched_ragged_streams(oracle, ctx, ans):
    import torch

    from test_decode_oracle_vs_ref import make_stream

    cb, per = oracle.capsule_bytes(ans), oracle.capsule_nodes(ans)
    n_streams, n_caps = 24, 304  # stride keeps every stream 16-byte aligned
    sync_every = lambda s: (90 + s) if s % 2 else None  # noqa: E731
    host = np.stack([make_stream(oracle, n_caps, 40.0 + s, seed=500 + s, sync_every=sync_every(s)) if ans == 0x85 else
                     make_capsules(oracle, ans, n_caps, 40.0 + s, seed=500 + s, sync_every=sync_every(s))
                     for s in range(n_streams)])
    counts_h = np.full(n_streams, n_caps, np.uint32)
    counts_h[3], counts_h[7], counts_h[11] = 123, 0, 1
    state_h = np.zeros((n_streams, 2), np.uint32)
    state_h[::3, 0] = 1
    state_h[1::4, 1] = 800
    dev = torch.device("cuda")
    caps = torch.from_numpy(host).to(dev)
    counts = torch.from_numpy(counts_h.view(np.int32)).to(dev)
    state = torch.from_numpy(state_h.view(np.int32)).to(dev)
    nodes = torch.zeros((n_streams, n_caps * per, 8), dtype=torch.uint8, device=dev)
    ncount = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    status = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
    state_out = torch.zeros((n_streams, 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_capsules_batch_dev(ans, caps.data_ptr(), counts.data_ptr(), n_streams, n_caps, 31, nodes.data_ptr(),
                                  ncount.data_ptr(), state_in=state.data_ptr(), capsule_status=status.data_ptr(),
                                  state_out=state_out.data_ptr())
    ctx.synchronize()
    torch.cuda.synchronize()
    hn = nodes.cpu().numpy().view(oracle.NODE_DTYPE).reshape(n_streams, n_caps * per)
    so = state_out.cpu().numpy().astype(np.uint32)
    for s in range(n_streams):
        k = int(counts_h[s])
        en, es, _, est = oracle.decode_capsules(ans, host[s, :k], 31, tuple(int(x) for x in state_h[s]))
        assert int(ncount[s]) == len(en)
        assert (hn[s, : len(en)].view(np.uint64) == en.view(np.uint64)).all()
        assert (status[s, :k].cpu().numpy().astype(np.uint32) == es).all()
        if ans in (0x85, 0x86):  # word 1, the last distance, is ultra-dense state: the dense decoder writes 0 there
            assert tuple(so[s]) == (est if ans == 0x86 else (est[0], 0))
