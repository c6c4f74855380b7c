"""Merged scans from the push (DESIGN.md 5.7.1 "Merged scans from the push"), a scan merger such as ira_laser_tools'
laserscan_multi_merger over the re-gridded LaserScans, restated on the CPU in numpy.  This docstring is the definition;
csrc/rescan.cu (merge_bins, rescan_hold_kernel, rescan_merge_dir_kernel, rescan_merge_kernel) computes the same bits.

M(settings, grids) is a pure function of one rpl_rescan_settings entry and a list of float32 rows of its grid
(ranges_size values each, oracle/rescan_oracle.py):

  M:      per bin, the least of the entry's seed (+inf with use_inf, else fl32(range_max + inf_epsilon)) and every
          row's value.  Re-grid values are never NaN and never -0, so the minimum does not depend on the order of the
          rows, and an empty list gives the seed in every bin.
  union:  Q keeps the least fl32(range) per bin whatever the point order, so for one entry and clouds c1..cn,
          M(settings, [Q(settings, c1), ..., Q(settings, cn)]) == Q(settings, c1 ++ ... ++ cn) bit for bit: the merge
          is pointcloud_to_laserscan over the concatenated clouds.

Session (the push form, rpl_capsule_stream_push_rescan_merge_msgs*; MergeModel restates it):

  groups: rpl_capsule_stream_set_rescan_merges puts each stream in at most one group g < n_groups, each with a
          max_age counted in merge pushes.  Refused, changing nothing: a group index neither below n_groups nor NONE,
          a group without a member, n_groups > n_streams, max_age > 65535.
  checks: a merge push is refused, changing nothing, unless every group's members have enabled entries equal in every
          field but pad and re-grid messages of one frame_id (the resolved target frame under
          RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS, else the LaserScan frame) -- checked at call time, since other set calls
          can change both after the groups are set.
  held:   after each merge push, a grouped stream s holds the ranges of the newest re-grid message of s the call wrote
          (size > 0: it fit rescans->capacity), as published (with a window, W's output), with that message's stamp
          and the call's number.  A call that wrote none of s's leaves s's held grid as it was.  (A window takes a
          re-grid that did not fit; a held grid is what a merger downstream received.)
  seq:    the number of merge pushes that succeeded, this one included.  Group g publishes one message in a call iff a
          member's held grid is from this call.  Its contributors are the members holding a grid with seq - held_seq
          <= max_age (0: this call only), so a stopped or dead lidar drops out after max_age calls.
  message: the re-grid message, byte for byte, of the contributor with the newest stamp ((sec, nanosec); a tie goes to
          the lowest stream index), with M over the contributors' held grids in place of its ranges.  Within one call
          every other byte is the same for every member, by the checks; a held grid from an earlier call keeps its
          message's header, which a call with or without RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS may have chosen.  One
          message per group per call: revolutions of different streams within one push have no order the call can
          observe.
  packing: merged is indexed by group; offsets the exclusive scan of the sizes each rounded up to 16; a message is
          written iff offset + size <= capacity, so the written messages are a prefix; total the end of the last.
  emptied: stream s's held grid, by session create; any set_rescan_merges call; set_rescans, set_rescan_windows or
          set_scan_cloud_transforms with s masked in; set_frames; reset with s masked in; an import into s; a switch of
          s's answer type.  A refused call changes no held grid and no seq; other calls neither read nor advance them.
"""
from __future__ import annotations

import numpy as np

from oracle import cdr_oracle as CDR
from oracle import rescan_oracle as RQ

NONE = 0xFFFFFFFF
MAX_AGE = 65535


def M(s, grids) -> np.ndarray:
    """the merged ranges of the rows `grids` of entry s: float32 [ranges_size]"""
    out = np.full(RQ.ranges_size(s), RQ.seed(s), np.float32)
    for g in grids:
        out = np.minimum(out, np.asarray(g, np.float32))
    return out


def merge_batch(s, rows, row_group, n_groups) -> np.ndarray:
    """rpl_rescan_merge_batch_dev: row g is M over the rows r with row_group[r] == g; rows of no group are not read"""
    rows = np.asarray(rows, np.float32).reshape(len(row_group), RQ.ranges_size(s))
    return np.array([M(s, [rows[r] for r in range(len(row_group)) if row_group[r] == g]) for g in range(n_groups)],
                    np.float32).reshape(n_groups, RQ.ranges_size(s))


def merges_ok(group_of_stream, max_age) -> bool:
    """the limits rpl_capsule_stream_set_rescan_merges enforces"""
    n_groups = len(max_age)
    if n_groups > len(group_of_stream) or any(a > MAX_AGE for a in max_age):
        return False
    if any(g != NONE and g >= n_groups for g in group_of_stream):
        return False
    return all(g in group_of_stream for g in range(n_groups))


def ranges_at(msg: bytes) -> tuple[int, int]:
    """(byte offset, count) of a re-grid message's ranges: the message ends with them and an empty intensities"""
    n = len(CDR.parse_laserscan(msg)["ranges"])
    return len(msg) - 4 - 4 * n, n


def stamp(msg: bytes) -> tuple[int, int]:
    m = CDR.parse_laserscan(msg)
    return m["sec"], m["nanosec"]


def pack(msgs, capacity):
    """(offsets, sizes, total) of merged messages by group (None: none) packed into `capacity` bytes"""
    sizes = [0 if m is None else len(m) for m in msgs]
    offsets, at = [], 0
    for n in sizes:
        offsets.append(at)
        at += (n + 15) // 16 * 16
    total = max([o + n for o, n in zip(offsets, sizes) if n] or [0])
    fits = [n > 0 and o + n <= capacity for o, n in zip(offsets, sizes)]
    return offsets, [n if f else 0 for n, f in zip(sizes, fits)], total


class MergeModel:
    """The session's merge state: groups, held grids (the held message, whose ranges are the grid) and seq"""

    def __init__(self, n_streams):
        self.n = n_streams
        self.groups = None  # None: before the first set_rescan_merges
        self.max_age = []
        self.held = [None] * n_streams  # (message bytes, seq)
        self.seq = 0

    def set_merges(self, group_of_stream, max_age):
        if not merges_ok(group_of_stream, max_age):
            return False
        self.groups = [list(np.flatnonzero(np.asarray(group_of_stream, np.int64) == g)) for g in range(len(max_age))]
        self.max_age = list(max_age)
        self.empty(None)
        return True

    def empty(self, mask):
        for s in range(self.n):
            if mask is None or mask[s]:
                self.held[s] = None

    def push(self, written, entry):
        """one merge push that succeeded: written[s] the re-grid messages of s the call wrote, in slot order;
        entry(s) stream s's settings.  Returns the merged message (bytes) or None per group."""
        assert self.groups is not None
        self.seq += 1
        for grp in self.groups:
            for s in grp:
                if written[s]:
                    self.held[s] = (written[s][-1], self.seq)
        out = []
        for g, grp in enumerate(self.groups):
            live = [s for s in grp if self.held[s] is not None and self.seq - self.held[s][1] <= self.max_age[g]]
            if not any(self.held[s][1] == self.seq for s in live):
                out.append(None)
                continue
            pick = max(live, key=lambda s: (stamp(self.held[s][0]), -s))  # newest stamp, then lowest index
            msg = self.held[pick][0]
            at, n = ranges_at(msg)
            grids = [np.frombuffer(self.held[s][0], np.float32, n, ranges_at(self.held[s][0])[0]) for s in live]
            out.append(msg[:at] + M(entry(pick), grids).tobytes() + msg[at + 4 * n:])
        return out
