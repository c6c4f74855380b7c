// rescan_args.h -- argument block of the re-gridding kernel (rescan.cu): pointcloud_to_laserscan's cloudCallback over
// the projected clouds, oracle/rescan_oracle.py's Q(settings, cloud) composed onto P and the transform rule.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "scan_cloud_args.h"

namespace rpl {

constexpr uint32_t kRescanMaxBins = 8192;  // a slot's grid, in shared memory

// one rpl_rescan_settings entry as the kernel reads it, resolved once on the host
struct RescanGrid {
  float angle_min, angle_max, angle_increment, range_min, range_max, min_height, max_height, scan_time;
  uint32_t seed;  // the float bits every beam starts at: +inf (use_inf) or fl32(range_max + inf_epsilon)
  uint32_t bins;  // ranges_size; 0 for a disabled entry (its slots have no message)
};

struct RescanArgs {
  // The projection whose points are re-gridded, as scan_cloud_kernel reads it: the slots' LaserScans (rows or a
  // session's work block), their window and cutoff, and, with c.transform, the stream's transform rows.  With c.m.out,
  // a session's messages: c.m.offsets / c.m.sizes place slot i's (size 0: none), with the header c.cloud_hdr
  // (c.transform) or c.m.hdr, and c.m's stamps.  c's tails and kept counts are not read.
  ScanCloudArgs c;
  const RescanGrid* grid;  // [n_slots / c.m.max_scans] a session's table; null: grid_one for every slot
  RescanGrid grid_one;
  float* out;              // rows: slot i's grid_one.bins ranges at out + i * grid_one.bins
};

cudaError_t launch_rescan(const RescanArgs& a, int num_sms, cudaStream_t stream);

// ---- windows over the re-gridded scans (oracle/rescan_window_oracle.py W; laser_filters' LaserArrayFilter) ----------
constexpr uint32_t kRescanWindowMax = 16;  // observations, and the values a bin's statistic takes, in registers
constexpr uint32_t kRescanWindowMedian = 0, kRescanWindowMean = 1;

// one stream's window as the kernel reads it: observations >= 2, its ring (observations - 1 rows of the stream's bins,
// row r's bin b at ring + r * bins + b) at the session ring's float offset `ring`
struct RescanWindow {
  unsigned long long ring;
  uint32_t observations, statistic;
};

// A push's windows over the chunk's streams that have one, one CTA per stream, behind rescan_kernel: r as rescan_kernel's
// push form (r.c reads the placed LaserScans; r.c.m.sizes are the re-grid messages' sizes, 0: not written; r.grid at
// the chunk's first stream).  Each of the stream's slots whose LaserScan message was written (r.c.scan_sizes[i] > 0),
// in slot order: the grid (the message's ranges, or built again when the message did not fit), then per bin W over the
// ring's values and the grid's, into the message; the grid goes into the ring.
struct RescanWindowArgs {
  RescanArgs r;
  const uint32_t* streams;    // [n] the session indices of the chunk's streams with a window
  uint32_t n, stream0;        // stream0: the chunk's first stream, so that streams[q] - stream0 counts from the chunk
  const RescanWindow* win;    // [streams] at the chunk's first stream
  uint2* state;               // [streams] at the chunk's first stream: {values held (<= observations - 1), next row}
  float* ring;
};
cudaError_t launch_rescan_window(const RescanWindowArgs& a, int num_sms, cudaStream_t stream);
// stateless: row t of out is W over rows max(0, t - observations + 1) .. t of in ([n_scans][bins])
cudaError_t launch_rescan_window_batch(const float* in, uint32_t n_scans, uint32_t bins, uint32_t observations,
                                       uint32_t statistic, float* out, int num_sms, cudaStream_t stream);

// ---- merged scans from the push (oracle/rescan_merge_oracle.py M; a scan merger over the re-gridded scans) ----------
constexpr uint32_t kRescanMergeNone = 0xFFFFFFFFu;  // a stream in no group, a row of no group

// A stream's held grid as the kernels keep it: its ranges in a row of kRescanMaxBins floats, the stamp of the re-grid
// message they came from, the merge push that wrote it (seq >= 1) and the header table that message took: hdr 0,
// nothing held; 1, the LaserScan frame's; 2, the target frame's (RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS).  The set calls
// that change either table empty the held grids, so the message is rebuilt byte for byte.
constexpr uint32_t kHeldScanHdr = 1, kHeldTargetHdr = 2;
struct RescanHeld {
  uint32_t sec, nanosec, seq, hdr;
};

// A push's held grids over the chunk's grouped streams, one CTA per stream, behind rescan_kernel and the window kernel:
// r as theirs (r.c.m.out / offsets / sizes / out_base: the re-grid messages as this chunk wrote them).  The newest slot
// of the stream whose re-grid message was written (size > 0) gives the held row its ranges and stamp.
struct RescanHoldArgs {
  RescanArgs r;
  const uint32_t* streams;  // [n] the session indices of the chunk's grouped streams
  uint32_t n, stream0;      // stream0: the chunk's first stream
  const uint32_t* row;      // [streams] at the chunk's first stream: the stream's held row
  RescanHeld* held;         // [streams] at the chunk's first stream
  float* rows;              // [held rows][kRescanMaxBins]
  uint32_t seq;             // this merge push's number
};
cudaError_t launch_rescan_hold(const RescanHoldArgs& a, int num_sms, cudaStream_t stream);

// The end of a merge push, over the session's groups: the directory (one CTA) decides each group's message, then the
// merge kernel (one CTA per message) writes it.  Group g's members are members[begin[g] .. begin[g + 1]) (session
// indices, ascending); a member contributes when it holds a grid of a push within max_age[g] of this one (seq -
// held.seq <= max_age[g]); the group publishes when a member's grid is from this push.  The message is the re-grid
// message of the contributor with the newest stamp (lowest index on a tie) -- the header its held grid took
// (hdr_scan or hdr_target, as RescanHeld::hdr says) with that stamp, then its entry's fields -- with M over the
// contributors' rows in place of its ranges.  Packed as the re-grid messages: offsets the exclusive scan of the sizes
// rounded up to 16, sizes[g] the size when it fits capacity (else 0), *total the end of the last.
struct RescanMergeArgs {
  const uint32_t *members, *begin, *max_age;
  uint32_t n_groups, seq;
  const uint32_t* row;                 // [n_streams]
  const RescanHeld* held;              // [n_streams]
  const float* rows;
  const StreamMsgHeader *hdr_scan, *hdr_target;  // [n_streams] each (hdr_target nullable: no transforms set)
  const RescanGrid* grid;              // [n_streams]
  uint32_t* pick;                      // [n_groups] the directory's choice for the merge kernel (kRescanMergeNone: none)
  unsigned long long capacity;
  unsigned long long *offsets, *total;  // offsets [n_groups]
  uint32_t* sizes;                      // [n_groups]
  unsigned long long* fit_end;          // nullable: the end of the last message that fits
  uint8_t* out;
};
cudaError_t launch_rescan_merge(const RescanMergeArgs& a, int num_sms, cudaStream_t stream);
// stateless: out[g] ([n_groups][bins]) is M over the rows r of in ([n_rows][bins]) with row_group[r] == g, from `seed`
cudaError_t launch_rescan_merge_batch(const float* in, const uint32_t* row_group, uint32_t n_rows, uint32_t n_groups,
                                      uint32_t bins, uint32_t seed, float* out, int num_sms, cudaStream_t stream);

}  // namespace rpl
