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

}  // namespace rpl
