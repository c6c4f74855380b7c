// scan_args.h -- argument block shared by the scan kernels and the C-ABI layer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lidar_args.h"

namespace rpl {

struct ScanBatchArgs {
  const uint2* nodes;      // [n_scans][stride] packed 8-byte nodes
  uint2* nodes_out;        // ascended nodes (nullable; must not alias nodes)
  const uint32_t* counts;  // [n_scans]
  uint32_t n_scans;
  uint32_t stride;
  float* ranges;           // [n_scans][stride] (nullable together with intensities)
  float* intensities;
  uint32_t* beam_counts;   // [n_scans] nullable
  float* angle_inc;        // [n_scans] nullable
  uint32_t* status;        // [n_scans] nullable
  uint32_t* path;          // [n_scans] nullable
  // fast kernel -> general kernel hand-off (device side, no host round trip)
  uint32_t* fallback_list;   // [n_scans]
  uint32_t* fallback_count;  // [1], zero when the fast kernel starts
  uint8_t is_new_protocol;
  uint8_t mode_a;
  uint8_t inverted;
  uint8_t apply_ascend;
  // PointCloud2 payload (extensions): when `xyzi` is set the kernels keep a node iff it is
  // measured AND range_min <= dist_m <= range_max AND intensity >= intensity_min, and write
  // (x, y, 0, intensity) at its rank among the kept nodes; beam_counts then holds the point count
  float4* xyzi;          // [n_scans][stride]
  const float2* trig;    // [65536] (cos, sin) of angle_rad(key)
  const float2* angle;   // [65536] (angle_rad, inverted angle): Mode A bins without FP64 on device
  float range_min, range_max, intensity_min;
  // scan views (rpl_scan_views_dev): when set, scan s is the `count` nodes starting at node `first` of the
  // whole `nodes` buffer -- views[s] = {first, count} -- instead of nodes[s * stride .. ) with counts[s];
  // outputs stay at s * stride.  nodes_total = nodes in the buffer (bulk copies must not run past it).
  const uint2* views;
  unsigned long long nodes_total;
  // per-stream settings (stream sessions, nullable): scan s takes is_new_protocol, inverted and (LaserScan) its Mode
  // A / Mode B from lidars[s / lidar_scans] instead of the fields above.  The shared-memory kernels are launched once
  // per mode in lidar_modes (bit 0 Mode B, bit 1 Mode A) and each serves its own mode's scans; the general kernel
  // takes every scan's mode from the table.
  const LidarSettings* lidars;
  uint32_t lidar_scans, lidar_modes;
  // placed ascended buffers (session nodes, nullable; the shared-memory EMIT kernels and the general kernel): scan s
  // writes its buffer at nodes_out + out_first[s] instead of nodes_out + s * stride.  An entry with kOutSkip set is
  // not this launch's scan: the kernels leave it before they read its nodes and write nothing for it, status included.
  // (The last member: the argument offsets of the kernels that do not read it stay what they were.)
  const unsigned long long* out_first;
  // placed LaserScan messages (a push's messages, rpl_capsule_stream_push_laserscan_msgs*; nullable; the shared-memory
  // MSG kernels and the general kernel): scan s writes its ranges at msg_out + msg_ranges[s] and its intensities 4 bytes
  // behind its last range, where the header writer puts the intensities count.  The payload is only 4-byte aligned (the
  // header's length follows the frame_id): the kernels store 4-byte words.  An entry with kOutSkip set has no message:
  // the kernels leave it as they leave an out_first skip.  (Behind out_first, for the same reason.)
  uint8_t* msg_out;
  const unsigned long long* msg_ranges;
  // per-stream clouds (RPL_CLOUD_PER_STREAM_CHAIN, nullable; the PointCloud2 payload of the shared-memory kernels and
  // the general kernel): scan s takes its window, and the fused kernel its SOR / voxel grid, from
  // clouds[s / lidar_scans] instead of the fields above and SmallArgs.  cloud_launches (bit 0 the window-only kernel,
  // bit 1 the fused kernel) tells which shared-memory launches the call makes: each serves the scans of its route
  // (cloud_route), a kCloudOff scan is the window-only launch's when it runs, else the fused one's, and is left with
  // point count 0 before its nodes are read.  (Behind msg_ranges, for the same reason.)
  const CloudSettings* clouds;
  uint32_t cloud_launches;
};
constexpr unsigned long long kOutSkip = 1ull << 63;

// per-CTA global workspace of the general kernel, sized for max_nodes
struct GeneralWorkspace {
  uint16_t* keyf;       // [ctas][max_nodes] final key of every node
  uint32_t* idx0;       // [ctas][max_nodes]
  uint32_t* idx1;       // [ctas][max_nodes]
  uint32_t* vidx;       // [ctas][max_nodes] sorted measured nodes -> buffer index
  unsigned long long* cell;  // [ctas][max_nodes] Mode A accumulators
  uint32_t max_nodes;
};

// per-CTA global scratch of the fast kernel (Mode A collision groups)
struct FastWorkspace {
  unsigned long long* group;  // [ctas][max_nodes] Mode A entries in bin-growth order (scan_fast.cu)
  uint32_t max_nodes;
};

// shared-memory-resident kernels (scan_small.cu): revolutions of at most kSmallMaxNodes nodes -- the SDK's own
// holder capacity -- for the LaserScan variants and the plain PointCloud2 projection; the PointCloud2 chain with
// SOR / voxel grid fused keeps (x, y), intensity and the cell accumulators in shared memory as well, which fits
// up to kSmallPostMaxNodes
constexpr uint32_t kSmallMaxNodes = 8192;
constexpr uint32_t kSmallPostMaxNodes = 4096;
struct SmallArgs {
  uint32_t cap;        // stride (or cap_nodes) rounded up to 64 nodes: capacity of the shared-memory arrays
  uint32_t max_nodes;  // the context's max_nodes (a larger count is a caller error)
  uint32_t use_tma;    // every scan base is 16-byte aligned: stage with one bulk-TMA copy
  uint32_t sor_k;      // PointCloud2 chain: 0 = no outlier removal
  float sor_alpha;
  float voxel;         // 0 = no voxel grid
};
bool scan_small_applies(uint32_t stride);
bool scan_small_post_applies(uint32_t stride);
cudaError_t scan_small_configure();
// a.xyzi set: PointCloud2 (window + xyz, then SOR / voxel grid in shared memory when asked for); else LaserScan
// Mode A/B with the ascended buffer when a.nodes_out is set.  Duplicate-key scans land in a.fallback_list.
// cap_nodes (PointCloud2 chain with SOR / voxel grid fused, scan views): size the shared-memory arrays for this many
// nodes instead of the stride; a view longer than that lands in a.fallback_list as well.  0: the stride.
cudaError_t launch_scan_small(const ScanBatchArgs& a, uint32_t max_nodes, uint32_t sor_k, float sor_alpha, float voxel,
                              int num_sms, cudaStream_t stream, uint32_t cap_nodes = 0);

constexpr int kFastThreads = 512;
constexpr int kGeneralThreads = 128;

cudaError_t launch_scan_fast(const ScanBatchArgs& a, const FastWorkspace& ws, int grid,
                             cudaStream_t stream);
// zero_next (nullable): [2] set to 0 by the kernel (the lane's next hand-off counter and scan ticket).  chained: launched as the
// programmatic dependent of the fast kernel before it on `stream`, which may trigger it early
// (griddepcontrol.launch_dependents).  stamp (nullable): the launch's profiling record (rpl_device.cuh stamp_start)
cudaError_t launch_scan_general(const ScanBatchArgs& a, const GeneralWorkspace& ws, int grid, bool all_scans,
                                uint32_t* zero_next, bool chained, unsigned long long* stamp, cudaStream_t stream);
size_t scan_fast_smem_bytes();
size_t scan_general_smem_bytes();
cudaError_t scan_fast_configure();     // opt-in dynamic shared memory, once per device
cudaError_t scan_general_configure();
int scan_fast_max_ctas_per_sm();
// v2: TMA-ring kernel (scan_tma.cu); needs 16-byte aligned scan bases
cudaError_t launch_scan_tma(const ScanBatchArgs& a, uint32_t max_nodes, int grid, cudaStream_t stream);
cudaError_t scan_tma_configure();
int scan_tma_max_ctas_per_sm(int mode);  // mode: 0 LaserScan Mode B, 1 Mode A, 2 PointCloud2
// LaserScan Mode B without the ascended buffer for strides in (kSmallMaxNodes, 32768]: each scan staged whole
// across a cluster of two CTAs (scan_tma.cu); 16-byte aligned scan bases, even grid of 2 x clusters
bool scan_tma_cluster_applies(uint32_t stride);
// ticket (nullable): a counter at zero from which the clusters draw scans at run time; without one each cluster takes
// a fixed share
cudaError_t launch_scan_tma_cluster(const ScanBatchArgs& a, uint32_t max_nodes, int grid, uint32_t* ticket,
                                    unsigned long long* stamp, cudaStream_t stream);
int scan_tma_max_clusters();  // two-CTA clusters of that kernel resident at once on the current device

}  // namespace rpl
