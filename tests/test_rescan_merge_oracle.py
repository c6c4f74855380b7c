"""CPU checks of oracle/rescan_merge_oracle.py, the definition of the merged scans: M of the members' grids is Q of the
concatenated clouds bit for bit, and the session model follows its publish, age, stamp and emptying rules over
scripted push histories."""
import math

import numpy as np
import pytest

from oracle import cdr_oracle as CDR
from oracle import rescan_merge_oracle as RM
from oracle import rescan_oracle as RQ
from oracle import rescan_window_oracle as RW


def _cloud(rng, n, s):
    """points around the sensor, a share on bin edges, out of the height band and out of the range window"""
    r = rng.uniform(0.0, 1.3 * min(s.range_max, 20.0), n)
    a = rng.uniform(-math.pi, math.pi, n)
    edge = rng.random(n) < 0.2  # exactly on a bin's lower edge
    k = rng.integers(0, max(RQ.ranges_size(s), 1), n)
    a[edge] = s.angle_min + k[edge] * s.angle_increment
    x, y = (r * np.cos(a)).astype(np.float32), (r * np.sin(a)).astype(np.float32)
    z = rng.uniform(-0.5, 0.8, n).astype(np.float32)
    return x, y, z


@pytest.mark.parametrize("use_inf", [True, False])
@pytest.mark.parametrize("grid", [(-math.pi, math.pi, math.pi / 180.0), (-1.0, 1.5, 0.01), (0.0, 0.5, 0.5 / 7)])
def test_merge_of_grids_is_the_grid_of_the_union(use_inf, grid):
    rng = np.random.default_rng(int(use_inf) + 10 * len(str(grid)))
    s = RQ.settings(*grid, range_min=0.2, range_max=9.0, min_height=-0.2, max_height=0.5, use_inf=use_inf,
                    inf_epsilon=0.7)
    for trial in range(12):
        n_clouds = int(rng.integers(1, 6))
        clouds = [_cloud(rng, int(rng.integers(0, 400)) if trial % 3 else 0, s) for _ in range(n_clouds)]
        grids = [RQ.regrid(s, *c) for c in clouds]
        union = RQ.regrid(s, *(np.concatenate([c[k] for c in clouds]) for k in range(3)))
        got = RM.M(s, grids)
        assert got.view(np.uint32).tolist() == union.view(np.uint32).tolist()
        assert RM.M(s, grids[::-1]).view(np.uint32).tolist() == union.view(np.uint32).tolist()
    assert (RM.M(s, []) == RQ.seed(s)).all()


def test_merge_batch_groups_rows():
    s = RQ.settings(0.0, 1.0, 0.25, range_max=5.0, use_inf=False, inf_epsilon=1.0)
    rows = np.array([[1, 7, 7, 2], [3, 1, 8, 8], [0.5, 0.5, 0.5, 0.5], [4, 4, 0.25, 9]], np.float32)
    got = RM.merge_batch(s, rows, [0, 0, RM.NONE, 2], 4)
    seed = np.float32(6.0)
    assert got.tolist() == [[1, 1, 6, 2], [seed] * 4, [4, 4, 0.25, 6], [seed] * 4]


def test_set_merges_limits():
    assert RM.merges_ok([0, 1, RM.NONE, 0], [0, 3])
    assert RM.merges_ok([RM.NONE] * 3, [])
    assert not RM.merges_ok([0, 2, 0], [0, 0])  # index not below n_groups
    assert not RM.merges_ok([0, 0, RM.NONE], [1, 1])  # group 1 is empty
    assert not RM.merges_ok([0], [1, 1])  # more groups than streams
    assert not RM.merges_ok([0, 1], [0, RM.MAX_AGE + 1])


S = RQ.settings(0.0, 1.0, 0.25, range_max=5.0, use_inf=True)
SCAL = (S.angle_min, S.angle_max, S.angle_increment, 0.0, S.scan_time, S.range_min, S.range_max)


def _msg(sec, nsec, ranges, frame="base_link"):
    return CDR.laserscan_cdr(sec, nsec, frame, SCAL, np.asarray(ranges, np.float32), np.zeros(0, np.float32))


def _ranges(msg):
    return CDR.parse_laserscan(msg)["ranges"].tolist()


def _push(m, written):
    w = [[] for _ in range(m.n)]
    for s, msgs in written.items():
        w[s] = list(msgs)
    return m.push(w, lambda s: S)


def test_publish_rule_contributors_and_ages():
    m = RM.MergeModel(5)
    assert m.set_merges([0, 0, 1, RM.NONE, 1], [0, 3])
    a, b, c, e = _msg(1, 0, [1, 9, 9, 9]), _msg(1, 5, [9, 2, 9, 9]), _msg(2, 0, [3, 3, 3, 3]), _msg(2, 1, [9, 9, 9, 1])
    out = _push(m, {0: [a], 1: [b], 2: [c], 3: [_msg(9, 9, [0, 0, 0, 0])]})
    assert _ranges(out[0]) == [1, 2, 9, 9]  # both members, this call
    assert CDR.parse_laserscan(out[0])["nanosec"] == 5  # b is the newer
    assert _ranges(out[1]) == [3, 3, 3, 3]  # the ungrouped stream 3 takes no part
    out = _push(m, {})  # nothing written: no group publishes, whatever it holds
    assert out == [None, None]
    out = _push(m, {0: [a]})  # max_age 0: only this call's grids
    assert _ranges(out[0]) == [1, 9, 9, 9] and out[1] is None
    out = _push(m, {4: [e]})  # max_age 3: stream 2's grid from three calls ago still counts
    assert _ranges(out[1]) == [3, 3, 3, 1] and CDR.parse_laserscan(out[1])["sec"] == 2
    assert CDR.parse_laserscan(out[1])["nanosec"] == 1
    out = _push(m, {4: [e]})  # four calls ago: stream 2 has dropped out
    assert _ranges(out[1]) == [9, 9, 9, 1]
    assert m.seq == 5


def test_max_age_one_and_idle_members():
    m = RM.MergeModel(3)
    m.set_merges([0, 0, 0], [1])
    g = [_msg(5, s, [s + 1.0] * 4) for s in range(3)]
    assert _ranges(_push(m, {0: [g[0]], 1: [g[1]]})[0]) == [1.0] * 4
    assert _ranges(_push(m, {2: [g[2]]})[0]) == [1.0] * 4  # 0 and 1 are one call old
    out = _push(m, {2: [g[2]]})
    assert _ranges(out[0]) == [3.0] * 4  # now two calls old: only stream 2
    assert _push(m, {}) == [None]


def test_newest_written_message_is_held_and_unfitting_ones_are_not():
    """the newest message the call wrote is held; a revolution whose re-grid message did not fit is not in `written`,
    so the stream keeps what it held (or its older message of the same call)"""
    m = RM.MergeModel(2)
    m.set_merges([0, 0], [5])
    old, new = _msg(1, 0, [4, 4, 4, 4]), _msg(3, 0, [2, 8, 8, 8])
    _push(m, {0: [old, new]})
    out = _push(m, {1: [_msg(2, 0, [8, 8, 8, 3])]})  # stream 0 wrote nothing: it still holds `new`
    assert _ranges(out[0]) == [2, 8, 8, 3] and CDR.parse_laserscan(out[0])["sec"] == 3


def test_windowed_members_contribute_their_published_ranges():
    m = RM.MergeModel(2)
    m.set_merges([0, 0], [0])
    raw = [np.array([1, 6, 6, 6], np.float32), np.array([5, 6, 6, 6], np.float32)]
    pub, held = RW.window_stream(2, RW.MEAN, raw)
    msgs = [_msg(1, k, p) for k, p in enumerate(pub)]
    out = _push(m, {0: [msgs[-1]], 1: [_msg(0, 0, [9, 9, 1, 9])]})
    assert _ranges(out[0]) == [3, 6, 1, 6]  # the mean (1 + 5) / 2, not the raw 5


def test_stamp_tie_goes_to_the_lowest_index_and_bytes_come_from_the_pick():
    m = RM.MergeModel(4)
    m.set_merges([RM.NONE, 0, 0, 0], [0])
    out = _push(m, {3: [_msg(7, 7, [1, 1, 1, 1], "f")], 1: [_msg(7, 7, [2, 2, 2, 2], "f")],
                    2: [_msg(7, 6, [3, 3, 3, 3], "f")]})
    want = _msg(7, 7, [1, 1, 1, 1], "f")
    assert out[0] == want  # stamps 7.7 tie between 1 and 3; every other byte is the same either way


def test_emptying():
    m = RM.MergeModel(3)
    m.set_merges([0, 0, 0], [9])
    _push(m, {s: [_msg(1, s, [s + 1.0] * 4)] for s in range(3)})
    m.empty([0, 1, 0])  # a masked emptying call: stream 1 only
    out = _push(m, {2: [_msg(2, 0, [9, 9, 9, 9])]})
    assert _ranges(out[0]) == [1, 1, 1, 1]
    m.empty(None)  # set_frames, or any set_rescan_merges call
    assert _push(m, {}) == [None]
    assert _ranges(_push(m, {1: [_msg(3, 0, [7, 7, 7, 7])]})[0]) == [7] * 4
    assert m.set_merges([0, 0, 0], [9])  # a new layout: every held grid empty
    assert all(h is None for h in m.held)
    assert not m.set_merges([0, 1, 1], [9])  # refused: nothing changes
    assert m.groups == [[0, 1, 2]]


def test_pack_is_a_prefix():
    msgs = [_msg(1, 0, [1] * 4), None, _msg(1, 0, [1] * 4, "longer_frame"), _msg(1, 0, [1] * 4)]
    offs, sizes, total = RM.pack(msgs, 10**6)
    assert offs[1] == offs[2] == (len(msgs[0]) + 15) // 16 * 16 and sizes[1] == 0
    assert total == offs[3] + len(msgs[3])
    _, cut, _ = RM.pack(msgs, total - 1)
    assert cut[:3] == sizes[:3] and cut[3] == 0
