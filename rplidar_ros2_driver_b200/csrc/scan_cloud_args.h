// scan_cloud_args.h -- argument block of the scan projection kernels (scan_cloud.cu): laser_geometry's projectLaser of
// published LaserScans, oracle/scan_cloud_oracle.py's P(params, scan).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cdr_args.h"

namespace rpl {

// the channel bits of rpl_scan_cloud_params (laser_geometry's ChannelOption): each adds one 4-byte field after x, y, z;
// the viewpoint (transforming calls only) adds three after those; kScanCloudPerStreamTransforms is an option
constexpr uint32_t kScanCloudIntensity = 0x01, kScanCloudIndex = 0x02, kScanCloudDistance = 0x04,
                   kScanCloudTimestamp = 0x08, kScanCloudChannels = 0x0F, kScanCloudViewpoint = 0x10,
                   kScanCloudPerStreamTransforms = 0x100;

// The PointCloud2 members between the header and the data (height .. data length) for one channel set: identical
// bytes for every frame id, as CloudTail.  ScanCloudTail: at most 192 bytes (x, y, z and all four channels);
// ScanCloudTailXf, a transforming call's: at most 264 (the viewpoint's three fields too)
template <uint32_t Words>
struct ScanCloudTailOf {
  uint32_t w[Words];
  uint32_t bytes;
  uint32_t at_width, at_row_step, at_data;  // word indices patched per message
};
using ScanCloudTail = ScanCloudTailOf<48>;
using ScanCloudTailXf = ScanCloudTailOf<66>;

struct ScanCloudArgs {
  // the LaserScans: m.counts (beams), m.ranges, m.intensities ([.][m.stride]), m.angle_increment over slots
  // [m.slot0, m.slot0 + m.n).  With m.out, a session's messages: m.hdr, stamps, m.lidars / m.mode_a give each slot's
  // header, range_max and time_increment as its LaserScan message carries them, m.offsets / m.sizes place it (size 0:
  // no message), and kept[i] is its point count.  Without: rows.
  MsgWriteArgs m;
  uint32_t channels, point_step;
  float range_cutoff;                // < 0: each scan's range_max
  float range_min, range_max;        // rows: every scan's (messages: kLaserScanRangeMin and the stream's range_max)
  const float* time_increment;       // rows: [n] nullable (0)
  uint32_t* kept;                    // [n_slots] the kept counts: the count pass writes them (rows: the write pass)
  float* points;                     // rows: scan s's records at points + s * m.stride * point_step / 4
  ScanCloudTail tail;                // messages
  // A push's LaserScans, read where its scan kernels wrote them (scan_msgs non-null; m.ranges, m.intensities unused):
  // slot i's ranges at scan_msgs + place[i], its intensities m.counts[i] + 1 floats later; a slot whose scan_sizes[i]
  // is 0 has no LaserScan message and no beams
  const uint8_t* scan_msgs;
  const unsigned long long* place;
  const uint32_t* scan_sizes;
  // A transforming call (transform != 0; DESIGN.md 5.7.1 "Projected clouds in a target frame"): slot i's stream's rows
  // {R_k0, R_k1, t_k, on} (k = 0, 1, 2) at xf + 3 * (i / m.max_scans), or xf_one when xf is null; on (row 0's w) is 0
  // for a disabled entry, whose points stay P's.  Messages take cloud_hdr's header ([n_slots / m.max_scans], the target
  // frame) and tail_xf; range_max still comes from m.hdr.  (Behind every other member: the calls without a transform
  // read the block as before.)
  uint32_t transform;
  const float4* xf;
  float4 xf_one[3];
  const StreamMsgHeader* cloud_hdr;
  ScanCloudTailXf tail_xf;
};

// the count pass: kept[i] of every slot [m.slot0, m.slot0 + m.n) (0 for a slot without beams)
cudaError_t launch_scan_cloud_count(const ScanCloudArgs& a, int num_sms, cudaStream_t stream);
// the write pass: rows (and kept[]), or the placed messages
cudaError_t launch_scan_cloud(const ScanCloudArgs& a, int num_sms, cudaStream_t stream);

}  // namespace rpl
