"""The numpy builder of the stream sessions' packed messages (rpl_*_stream_{laserscan,cloud}_msgs*), which the GPU tests
hold the device bytes against: the header scalars of one scan from its begin / end stamps, the messages
(oracle/cdr_oracle.py's writers) and their packing.  Checked here against a message laid out by hand and against the
stamp and period rules on hand-picked values."""
import struct

import numpy as np
import pytest

from oracle.cdr_oracle import laserscan_cdr, parse_laserscan, parse_pointcloud2, pointcloud2_cdr

TWO_PI_F32 = np.float32(2.0 * np.pi)
RANGE_MIN = np.float32(0.15)
INT32_MAX = 2 ** 31 - 1


def _i64(v):
    """v as int64, two's complement"""
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


def msg_stamp(b_us, clock_offset_ns):
    """header.stamp of a scan-begin stamp (SDK us) on the caller's clock: (sec, nanosec), (0, 0) when b_us is 0, the
    time is negative or sec does not fit int32"""
    if b_us == 0:
        return 0, 0
    t = _i64(int(b_us) * 1000 + int(clock_offset_ns))
    if t < 0:
        return 0, 0
    sec, nsec = divmod(t, 10 ** 9)
    if sec > INT32_MAX:
        return 0, 0
    return sec, nsec


def scan_period(b_us, e_us):
    """rclcpp Duration::seconds() of the stamp-to-stamp period, 0.0 when a stamp is unknown or e <= b"""
    if b_us == 0 or e_us == 0 or e_us <= b_us:
        return 0.0
    return float(_i64((int(e_us) - int(b_us)) * 1000)) / 1e9


def laserscan_scalars(b_us, e_us, beams, mode_a, angle_increment, range_max):
    """angle_min, angle_max, angle_increment, time_increment, scan_time, range_min, range_max"""
    d = scan_period(b_us, e_us)
    denom = float(beams) if mode_a else float(max(beams - 1, 1))
    return [np.float32(0.0), TWO_PI_F32, np.float32(angle_increment), np.float32(d / denom), np.float32(d), RANGE_MIN,
            np.float32(range_max)]


def expected_laserscan(frame_id, range_max, b_us, e_us, clock_offset_ns, mode_a, ranges, intensities, angle_increment):
    """the message of one slot, None when the scan has no beams"""
    n = len(ranges)
    if n == 0:
        return None
    sec, nsec = msg_stamp(b_us, clock_offset_ns)
    return laserscan_cdr(sec, nsec, frame_id, laserscan_scalars(b_us, e_us, n, mode_a, angle_increment, range_max),
                         ranges, intensities)


def expected_cloud(frame_id, b_us, clock_offset_ns, xyzi):
    sec, nsec = msg_stamp(b_us, clock_offset_ns)
    return pointcloud2_cdr(sec, nsec, frame_id, xyzi)


def pack(msgs):
    """msgs: per slot bytes or None -> (offsets, sizes, total): each message at a multiple of 16, offsets the exclusive
    scan of the sizes rounded up to 16, total the end of the last message"""
    offs, sizes, at, total = [], [], 0, 0
    for m in msgs:
        s = 0 if m is None else len(m)
        offs.append(at)
        sizes.append(s)
        if s:
            total = at + s
        at += (s + 15) // 16 * 16
    return np.array(offs, np.uint64), np.array(sizes, np.uint32), total


def packed_bytes(msgs):
    """the packed buffer up to the end of the last message (padding zero)"""
    offs, sizes, total = pack(msgs)
    buf = bytearray(total)
    for m, o in zip(msgs, offs.tolist()):
        if m is not None:
            buf[o: o + len(m)] = m
    return bytes(buf)


# ---- the builder against a message laid out by hand ------------------------------------------------------------------
def _hand_laserscan():
    """frame_id "base_scan_7" (11 characters: length 12 with the NUL, no padding after it), stamp 1700000123.000456789
    from B = 1_700_000_123_000_456 us + 789 ns, a 0.1 s period over 3 beams in Mode B"""
    b = bytearray(b"\x00\x01\x00\x00")
    b += struct.pack("<iI", 1700000123, 456789)
    b += struct.pack("<I", 12) + b"base_scan_7\x00"
    d = 0.1
    b += struct.pack("<7f", 0.0, float(np.float32(2 * np.pi)), 0.25, float(np.float32(d / 2)), float(np.float32(d)),
                     0.15, 16.5)
    b += struct.pack("<I3f", 3, 1.0, 2.0, float("inf"))
    b += struct.pack("<I3f", 3, 47.0, 0.0, 12.0)
    return bytes(b)


def test_builder_matches_hand_laid_laserscan():
    got = expected_laserscan("base_scan_7", 16.5, 1_700_000_123_000_456, 1_700_000_123_100_456, 789, False,
                             np.array([1.0, 2.0, np.inf], np.float32), np.array([47.0, 0.0, 12.0], np.float32), 0.25)
    assert got == _hand_laserscan()
    m = parse_laserscan(got)
    assert (m["sec"], m["nanosec"], m["frame_id"]) == (1700000123, 456789, "base_scan_7")


def test_builder_matches_hand_laid_pointcloud2():
    """frame_id "lidar" (5 characters + NUL, 2 bytes of padding), 2 points"""
    pts = np.array([[1, 2, 3, 4], [-1, -2, 0.5, 9]], np.float32)
    b = bytearray(b"\x00\x01\x00\x00") + struct.pack("<iI", 12, 3000) + struct.pack("<I", 6) + b"lidar\x00\x00\x00"
    b += struct.pack("<III", 1, 2, 4)
    for k, name in enumerate((b"x", b"y", b"z")):
        b += struct.pack("<I", 2) + name + b"\x00\x00\x00" + struct.pack("<I", 4 * k) + b"\x07\x00\x00\x00" + \
            struct.pack("<I", 1)
    b += struct.pack("<I", 10) + b"intensity\x00\x00\x00" + struct.pack("<I", 12) + b"\x07\x00\x00\x00" + \
        struct.pack("<I", 1)
    b += b"\x00\x00\x00\x00" + struct.pack("<III", 16, 32, 32) + pts.tobytes() + b"\x01"
    got = expected_cloud("lidar", 12_000_005, -2000, pts)  # 12.000005 s - 2 us
    assert got == bytes(b)
    assert parse_pointcloud2(got)["width"] == 2


# ---- stamps ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b_us, off, exp", [
    (0, 123, (0, 0)),                                        # unknown begin
    (1, 0, (0, 1000)),
    (1_000_000, -1, (0, 999_999_999)),                       # negative offset borrows from the seconds
    (2_500_000, -500_000_000, (2, 0)),
    (1_999_999, 1_000, (2, 0)),                              # nanoseconds wrap into the next second
    (1_999_999, 999, (1, 999_999_999)),
    (5, -5001, (0, 0)),                                      # t < 0
    (5, -5000, (0, 0)),                                      # t == 0: a representable stamp, which is {0, 0}
    (INT32_MAX * 1_000_000 + 999_999, 999, (INT32_MAX, 999_999_999)),
    (INT32_MAX * 1_000_000 + 999_999, 1000, (0, 0)),         # sec > INT32_MAX
    (10 ** 6, -(10 ** 18), (0, 0)),
])
def test_stamp_split(b_us, off, exp):
    assert msg_stamp(b_us, off) == exp


def test_period_rules():
    assert scan_period(0, 100) == 0.0 and scan_period(100, 0) == 0.0
    assert scan_period(100, 100) == 0.0 and scan_period(100, 99) == 0.0
    assert scan_period(1_000_000, 1_100_000) == 0.1
    assert scan_period(7, 7 + 123_457) == 123_457_000 / 1e9


@pytest.mark.parametrize("mode_a", [True, False])
def test_time_increment_rounding(mode_a):
    """time_increment is the double quotient rounded once to float32, not scan_time (already float32) divided"""
    b, e = 1_000_000, 1_000_000 + 133_337
    d = 133_337_000 / 1e9
    for beams in (1, 2, 3, 719, 1440, 3200):
        denom = beams if mode_a else max(beams - 1, 1)
        s = laserscan_scalars(b, e, beams, mode_a, 0.01, 12.0)
        assert s[4] == np.float32(d)
        assert s[3] == np.float32(d / denom)
    assert laserscan_scalars(0, e, 10, mode_a, 0.01, 12.0)[3:5] == [0.0, 0.0]


def test_mode_b_single_beam_divides_by_one():
    s = laserscan_scalars(10, 10 + 50_000, 1, False, 0.0, 12.0)
    assert s[3] == s[4] == np.float32(0.05)


def test_packing():
    msgs = [b"a" * 17, None, b"b" * 16, b"c" * 1, None]
    offs, sizes, total = pack(msgs)
    assert offs.tolist() == [0, 32, 32, 48, 64] and sizes.tolist() == [17, 0, 16, 1, 0] and total == 49
    buf = packed_bytes(msgs)
    assert len(buf) == 49 and buf[32:48] == b"b" * 16 and buf[17:32] == bytes(15)
    offs, sizes, total = pack([None, None])
    assert offs.tolist() == [0, 0] and sizes.tolist() == [0, 0] and total == 0
