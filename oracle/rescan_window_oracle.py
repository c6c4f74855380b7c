"""Windows over the re-gridded LaserScans (DESIGN.md 5.7.1 "Windows over the re-gridded scans"), laser_filters'
LaserArrayFilter with MultiChannelMedianFilterFloat or MultiChannelMeanFilterFloat, restated on the CPU in numpy.  This
docstring is the definition; csrc/rescan.cu (window_stat) computes the same bits.

W(window, xs) is a pure function of a non-empty list xs of float32 rows of one stream's grid (Q's ranges, oracle/
rescan_oracle.py), oldest first, with n = len(xs) <= window.observations:

  median: per bin, the element of rank (n - 1) // 2 of the n values in ascending order -- for even n the lower median.
          This is what the filters package's median() returns (kth_smallest with n/2 or n/2 - 1).
  mean:   per bin, a float32 sum from +0.0, oldest to newest, rounded at each step, then fl32(sum / n).
  values: re-grid values are never NaN and never -0: they are finite, +inf, or the entry's seed range_max +
          inf_epsilon.  So the median is one of the values, whatever the selection algorithm, and the device equals this
          restatement bit for bit.  A +inf seed takes part like any other value, as it would downstream of
          pointcloud_to_laserscan.
  limits: 1 <= observations <= 16 (1: no window, W is the newest row), statistic 0 (median) or 1 (mean); anything else
          is refused (RPL_RESULT_INVALID_DATA).

Stream window (the session's push form, rpl_capsule_stream_push_rescan_msgs*): stream s's window is the sequence of the
stream's raw re-gridded scans that qualify, newest last.  A revolution qualifies when a push-form call returned it, its
LaserScan message was written (scans->msg_sizes[i] > 0) and the stream's re-grid entry is enabled.  The message of
revolution k carries W(window, the last min(observations, k) entries) in place of Q's ranges; every other byte is Q's
message (header, the newest revolution's stamp, frame, angles, sizes), as LaserArrayFilter republishes scan_in.
window_stream below restates it over the sequence of qualifying grids.

The package's loops are restated from memory of its source, which was not at hand when this was written (as in
oracle/rescan_oracle.py): these bytes are the definition either way.
"""
from __future__ import annotations

import numpy as np

MEDIAN, MEAN = 0, 1
MAX_OBSERVATIONS = 16


def window_ok(observations: int, statistic: int) -> bool:
    """the limits of a window"""
    return 1 <= observations <= MAX_OBSERVATIONS and statistic in (MEDIAN, MEAN)


def W(statistic: int, xs) -> np.ndarray:
    """the statistic of the rows xs (oldest first, each [bins] float32), per bin"""
    a = np.asarray(xs, dtype=np.float32)
    assert a.ndim == 2 and a.shape[0] >= 1
    n = a.shape[0]
    if statistic == MEDIAN:
        return np.sort(a, axis=0, kind="stable")[(n - 1) // 2].copy()
    assert statistic == MEAN
    s = np.zeros(a.shape[1], np.float32)  # +0.0
    with np.errstate(over="ignore"):
        for row in a:
            s = (s + row).astype(np.float32)  # float32 + float32: rounded at each step
        return (s / np.float32(n)).astype(np.float32)


def window_batch(observations: int, statistic: int, rows) -> np.ndarray:
    """rpl_rescan_window_batch_dev: row t is W over rows max(0, t - observations + 1) .. t (an empty window at row 0)"""
    a = np.asarray(rows, dtype=np.float32)
    out = np.empty_like(a)
    for t in range(a.shape[0]):
        out[t] = W(statistic, a[max(0, t - observations + 1): t + 1])
    return out


def window_stream(observations: int, statistic: int, grids, start=()):
    """the ranges the push form publishes for the qualifying grids (oldest first) of one stream, whose window held
    `start` (oldest first) before them; returns (the published rows, the window after them)"""
    held = [np.asarray(g, np.float32) for g in start][-(observations - 1):] if observations > 1 else []
    out = []
    for g in grids:
        g = np.asarray(g, np.float32)
        out.append(W(statistic, held + [g]))
        held = (held + [g])[-(observations - 1):] if observations > 1 else []
    return out, held
