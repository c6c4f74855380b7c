"""GPU tests of the dense-capsule decoder (SURVEY.md 8(f) rank 1) against the restatement, which
tests/test_decode_oracle_vs_ref.py pins against the SDK's own unpacker.  Integer work: bit-exact."""
import numpy as np
import pytest

from test_decode_oracle_vs_ref import make_stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


@pytest.fixture(scope="module")
def ctx(R):
    c = R.Context(0, 40000, 64)
    yield c
    c.close()


def check(R, O, ctx, caps, sample_us=31, state=0):
    en, es, eo, estate = O.dense_decode(caps, sample_us, state)
    gn, gs, go, gstate = ctx.decode_dense(caps, sample_us, state)
    assert len(gn) == len(en)
    assert (gn.view(np.uint64) == en.view(np.uint64)).all()
    assert (gs == es).all() and (go == eo).all() and gstate == estate
    return gn, gs, gstate


@pytest.mark.parametrize("n_caps", [1, 2, 3, 255, 256, 257, 513, 2000])
def test_clean_streams_across_tile_boundaries(R, oracle, ctx, n_caps):
    check(R, oracle, ctx, make_stream(oracle, n_caps, 80.0, seed=n_caps))
    check(R, oracle, ctx, make_stream(oracle, n_caps, 80.0, seed=n_caps, sync_every=80), state=1)


def test_errors_sync_capsules_and_jumps(R, oracle, ctx):
    rng = np.random.default_rng(5)
    caps = make_stream(oracle, 900, 80.0, seed=1, sync_every=80)
    caps[rng.choice(900, 40, replace=False), 10] ^= 0x40
    caps[254:259, 2] ^= 0xFF  # checksum errors right on a tile boundary
    jump = make_stream(oracle, 50, 80.0, seed=2, start_deg=123.0)
    allc = np.concatenate([caps[:300], jump, caps[300:]])
    allc[511, 0] = 0x30  # bad sync nibble: reported, decoding goes on
    _, st, _ = check(R, oracle, ctx, allc)
    assert ((st & R.capi.CAPSULE_BAD_FRAME) != 0).sum() == 1
    assert ((st & R.capi.CAPSULE_CHECKSUM_ERR) != 0).sum() >= 40


@pytest.mark.parametrize("sample_us", [31, 63, 125, 476])
def test_jump_threshold(R, oracle, ctx, sample_us):
    for cpr in (80.0, 12.0, 5.0):
        check(R, oracle, ctx, make_stream(oracle, 300, cpr, seed=sample_us), sample_us=sample_us)


def test_sync_bit_alternation_and_state(R, oracle, ctx):
    q6 = (np.arange(700) % 3).astype(np.uint32)
    caps = oracle.make_dense_capsules(q6, np.zeros(700, bool), np.full((700, 40), 1234))
    for state in (0, 1):
        nodes, _, _ = check(R, oracle, ctx, caps, state=state)
        assert 0 < int((nodes["flag"] & 1).sum()) < len(nodes)


def test_random_streams(R, oracle, ctx):
    rng = np.random.default_rng(78)
    for t in range(30):
        n = int(rng.integers(1, 700))
        caps = make_stream(oracle, n, float(rng.uniform(4, 200)), seed=2000 + t,
                           sync_every=int(rng.integers(5, 100)) if t % 2 else None)
        for j in rng.choice(n, max(1, n // 20), replace=False):
            caps[j, int(rng.integers(2, 84))] ^= int(rng.integers(1, 256))
        check(R, oracle, ctx, caps, sample_us=int(rng.choice([31, 63, 125])), state=t & 1)


def test_batched_streams_and_chain_into_the_scan_path(R, oracle, ctx):
    """64 streams decoded in one launch; the decoded nodes of one revolution then go through the
    hot path and must give the same LaserScan as the CPU chain decode -> ascend -> publish."""
    import torch

    n_streams, n_caps = 64, 400
    host = np.stack([make_stream(oracle, n_caps, 80.0, seed=300 + s, sync_every=80) for s in range(n_streams)])
    dev = torch.device("cuda")
    caps = torch.from_numpy(host).to(dev)
    counts = torch.full((n_streams,), n_caps, dtype=torch.int32, device=dev)
    counts[3] = 123  # ragged
    sync_h = (np.arange(n_streams) % 3 == 0).astype(np.uint32)  # one state word per stream
    sync_in = torch.from_numpy(sync_h.view(np.int32)).to(dev)
    sync_out = torch.full((n_streams,), 7, dtype=torch.int32, device=dev)
    nodes = torch.zeros((n_streams, n_caps * 40, 8), dtype=torch.uint8, device=dev)
    ncount = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    status = torch.zeros((n_streams, n_caps), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # buffers were filled on torch's stream; the library runs on its own
    ctx.decode_dense_batch_dev(caps.data_ptr(), counts.data_ptr(), n_streams, n_caps, 31, nodes.data_ptr(),
                               ncount.data_ptr(), sync_state_in=sync_in.data_ptr(), capsule_status=status.data_ptr(),
                               sync_state_out=sync_out.data_ptr())
    ctx.synchronize()
    torch.cuda.synchronize()
    hn = nodes.cpu().numpy().view(oracle.NODE_DTYPE).reshape(n_streams, n_caps * 40)
    so = sync_out.cpu().numpy().astype(np.uint32)
    for s in range(n_streams):
        k = int(counts[s])
        en, es, _, est = oracle.dense_decode(host[s, :k], 31, int(sync_h[s]))
        assert int(ncount[s]) == len(en)
        assert (hn[s, : len(en)].view(np.uint64) == en.view(np.uint64)).all()
        assert (status[s, :k].cpu().numpy().astype(np.uint32) == es).all()
        assert int(so[s]) == est
    # one revolution of stream 0: nodes between the first two scan-start flags
    en, _, _, _ = oracle.dense_decode(host[0], 31, 0)
    starts = np.flatnonzero(en["flag"] & 1)
    rev = en[starts[0]: starts[1]]
    got = ctx.scan(rev.view(R.NODE_DTYPE), R.scan_params(1, 0, 0, 1))
    rc, asc = oracle.ascend(rev)
    hdr, r, it = oracle.publish(asc, oracle.scan_params(1, 0, 0, 1, 40.0, 0.1))
    assert got["beam_count"] == hdr.beam_count
    assert (got["ranges"].view(np.uint32) == r.view(np.uint32)).all()
