// scan_filter_args.h -- the LaserScan filter chain (scan_filter.cu; DESIGN.md 5.7.1 "LaserScan filters"): one entry as
// the kernel reads it, and the argument block of the kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {

constexpr uint32_t kScanFilterMaxWindow = 16;
constexpr uint32_t kScanFilterMaxBeams = 8192;
constexpr uint32_t kFootprintMaxPolygons = 4;
constexpr uint32_t kFootprintMaxVertices = 16;

// rpl_scan_filter_settings as stored: the same layout, but shadow_angle replaced by tan(shadow_angle) (double on the
// host, rounded to float) and `enabled` widened to a word
struct ScanFilter {
  float mask_lo[4], mask_hi[4];
  float range_lo, range_hi, intensity_min, speckle_max_diff, shadow_tan;
  uint32_t speckle_window, speckle_min_neighbours, shadow_window;
  uint32_t enabled;
};

// rpl_scan_footprint as the kernel reads it: the used polygons first (n_polygons of them), their vertices moved into
// the scan frame on the host (oracle/scan_footprint_oracle.py scan_frame); n_polygons 0: no footprint
struct ScanFootprint {
  float x[kFootprintMaxPolygons][kFootprintMaxVertices], y[kFootprintMaxPolygons][kFootprintMaxVertices];
  uint32_t n_vertices[kFootprintMaxPolygons];
  uint32_t invert[kFootprintMaxPolygons];
  uint32_t n_polygons;
};

// Scans [0, n_scans), each filtered in place with filters[s / per_filter] (or `one`) and the footprint
// footprints[s / per_filter] (or `one_footprint`):
//   rows (msg_out null): ranges + s * stride, intensities + s * stride;
//   placed messages (msg_out set): ranges at msg_out + place[s] (4-byte aligned), intensities M + 1 floats behind
//   them; an entry with kOutSkip set has no message and is left alone.
// M = beam_counts[s] (<= kScanFilterMaxBeams), the increment angle_increment[s].
struct ScanFilterArgs {
  const ScanFilter* filters;  // [n_scans / per_filter] device; nullptr: every scan takes `one`
  uint32_t per_filter;
  ScanFilter one;
  const ScanFootprint* footprints;  // [n_scans / per_filter] device; nullptr: every scan takes `one_footprint`
  ScanFootprint one_footprint;
  float* ranges;
  const float* intensities;
  uint32_t stride;
  uint8_t* msg_out;
  const unsigned long long* place;
  const uint32_t* beam_counts;
  const float* angle_increment;
  uint32_t n_scans;
};
cudaError_t launch_scan_filter(const ScanFilterArgs& a, int num_sms, cudaStream_t stream);

}  // namespace rpl
