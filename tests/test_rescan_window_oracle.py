"""CPU checks of oracle/rescan_window_oracle.py, the definition of the windows over the re-gridded LaserScans: the
median against an independent rank statement, the mean against float64 and a sequential float32 loop, over the
warm-up, even and odd counts, ties, +inf and seed values, and every limit."""
import numpy as np
import pytest

from oracle import rescan_window_oracle as RW

SEED = np.float32(np.float32(12.0) + np.float32(1.0))  # a range_max + inf_epsilon seed


def _rows(rng, n, bins, ties=False, specials=False):
    a = rng.uniform(0.05, 30.0, (n, bins)).astype(np.float32)
    if ties:
        a = np.round(a).astype(np.float32)  # few distinct values per bin
    if specials:
        m = rng.random((n, bins))
        a[m < 0.2] = np.inf
        a[(m >= 0.2) & (m < 0.35)] = SEED
    return a


def _check_median(xs, got):
    n = xs.shape[0]
    k = (n - 1) // 2
    for b in range(xs.shape[1]):
        col, v = xs[:, b], got[b]
        assert (col.view(np.uint32) == v.view(np.uint32)).any(), "the median is one of the inputs"
        assert int((col < v).sum()) <= k, "at most k inputs are strictly less"
        assert int((col <= v).sum()) >= k + 1, "at least k + 1 inputs are less or equal"


@pytest.mark.parametrize("n", list(range(1, 17)))
@pytest.mark.parametrize("kind", ["plain", "ties", "specials"])
def test_median_is_the_rank_statement(n, kind):
    rng = np.random.default_rng(1000 * n + len(kind))
    xs = _rows(rng, n, 97, ties=kind == "ties", specials=kind == "specials")
    got = RW.W(RW.MEDIAN, xs)
    assert got.dtype == np.float32 and got.shape == (97,)
    _check_median(xs, got)


def test_median_even_is_the_lower_median():
    xs = np.array([[4.0], [1.0], [3.0], [2.0]], np.float32)
    assert RW.W(RW.MEDIAN, xs)[0] == 2.0
    assert RW.W(RW.MEDIAN, xs[:3])[0] == 3.0
    assert RW.W(RW.MEDIAN, np.array([[np.inf], [5.0]], np.float32))[0] == 5.0
    assert RW.W(RW.MEDIAN, np.array([[np.inf], [5.0], [np.inf]], np.float32))[0] == np.inf


def _sequential_mean(col):
    s = np.float32(0.0)
    for v in col:
        s = np.float32(s + np.float32(v))
    return np.float32(s / np.float32(len(col)))


@pytest.mark.parametrize("n", list(range(1, 17)))
def test_mean_is_the_float32_loop_and_near_float64(n):
    rng = np.random.default_rng(n)
    xs = _rows(rng, n, 61)
    got = RW.W(RW.MEAN, xs)
    seq = np.array([_sequential_mean(xs[:, b]) for b in range(61)], np.float32)
    assert (got.view(np.uint32) == seq.view(np.uint32)).all()
    ref = xs.astype(np.float64).mean(axis=0)
    assert np.allclose(got, ref, rtol=1e-6, atol=0)


def test_mean_with_inf_and_seed():
    xs = np.array([[1.0, SEED, 2.0], [np.inf, SEED, 4.0]], np.float32)
    got = RW.W(RW.MEAN, xs)
    assert got[0] == np.inf and got[1] == SEED and got[2] == 3.0


def test_mean_overflow_is_inf_as_float32():
    big = np.float32(3.0e38)
    got = RW.W(RW.MEAN, np.array([[big], [big], [big]], np.float32))
    assert got[0] == np.inf  # the running float sum overflows, as the device's does


@pytest.mark.parametrize("obs", [1, 2, 3, 5, 8, 16])
@pytest.mark.parametrize("stat", [RW.MEDIAN, RW.MEAN])
def test_batch_warm_up_and_steady_state(obs, stat):
    rng = np.random.default_rng(obs * 7 + stat)
    rows = _rows(rng, 25, 33, specials=True)
    out = RW.window_batch(obs, stat, rows)
    for t in range(25):
        lo = max(0, t - obs + 1)
        exp = RW.W(stat, rows[lo: t + 1])
        assert (out[t].view(np.uint32) == exp.view(np.uint32)).all()
    if obs == 1:
        assert (out.view(np.uint32) == rows.view(np.uint32)).all()


@pytest.mark.parametrize("obs", [1, 2, 4, 16])
def test_stream_window_is_the_batch_across_splits(obs):
    rng = np.random.default_rng(obs)
    rows = _rows(rng, 30, 17, ties=True)
    whole = RW.window_batch(obs, RW.MEDIAN, rows)
    held, got = [], []
    for a, b in ((0, 3), (3, 4), (4, 20), (20, 30)):
        out, held = RW.window_stream(obs, RW.MEDIAN, rows[a:b], held)
        got += out
    assert (np.array(got).view(np.uint32) == whole.view(np.uint32)).all()
    assert len(held) == min(obs - 1, 30)


def test_limits():
    assert RW.window_ok(1, 0) and RW.window_ok(16, 1)
    assert not RW.window_ok(0, 0) and not RW.window_ok(17, 0) and not RW.window_ok(2, 2)
