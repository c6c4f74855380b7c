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

}  // namespace rpl
