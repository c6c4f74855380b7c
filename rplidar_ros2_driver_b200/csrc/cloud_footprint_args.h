// cloud_footprint_args.h -- the footprint pass of the PointCloud2 chain (cloud_footprint.cu; DESIGN.md 5.7.1
// "Footprints in the clouds"): the argument block of its kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lidar_args.h"
#include "scan_filter_args.h"

namespace rpl {

// Scans [0, n_scans) of per-scan clouds xyzi + s * stride with point_counts[s] points each, as steps 1-3 of the cloud
// chain leave them (angle order, before SOR and the voxel grid): the points scan s's footprint removes are dropped in
// place, the others keep their order, and point_counts[s] becomes the number kept.  Scan s takes footprints[s / per]
// (or `one`), its vertices in the scan frame; with lidars, a scan whose stream is inverted tests its points against
// the vertices (u, -v), since the cloud is not mirrored as the LaserScan is.
struct CloudFootprintArgs {
  float4* xyzi;
  uint32_t* point_counts;
  uint32_t n_scans, stride;
  const ScanFootprint* footprints;  // [n_scans / per] device; nullptr: every scan takes `one`
  const LidarSettings* lidars;      // [n_scans / per] device; nullptr: no scan is mirrored
  uint32_t per;
  ScanFootprint one;
};
cudaError_t launch_cloud_footprint(const CloudFootprintArgs& a, int num_sms, cudaStream_t stream);

}  // namespace rpl
