// scan_cloud_point.cuh -- which beams of a slot the projection keeps and where their points go, shared by the scan
// projection (scan_cloud.cu) and the scans re-gridded from it (rescan.cu), so that a re-gridded scan tests exactly the
// points the projected cloud publishes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "msg_fixed.cuh"
#include "scan_cloud_args.h"

namespace rpl {
namespace {

__device__ __forceinline__ bool keep_beam(float r, float range_min, float cutoff) {
  return r >= range_min && r < cutoff;  // NaN never, +inf never (cutoff <= +inf)
}

// the window of slot i: a session's LaserScan range_min and its stream's range_max, or the call's; the cutoff
__device__ __forceinline__ void slot_window(const ScanCloudArgs& a, uint32_t i, float* lo, float* cut) {
  const float hi = a.m.hdr ? a.m.hdr[i / a.m.max_scans].range_max : a.range_max;
  *lo = a.m.hdr ? kLaserScanRangeMin : a.range_min;
  *cut = a.range_cutoff >= 0.0f ? a.range_cutoff : hi;
}

// slot i's beams: its row, or its placed LaserScan message (a push's, 4-byte aligned: the loads stay 4-byte)
struct SlotBeams {
  uint32_t M;
  const float *rg, *ig;
};
__device__ __forceinline__ SlotBeams slot_beams(const ScanCloudArgs& a, uint32_t i) {
  if (!a.scan_msgs)
    return SlotBeams{min(a.m.counts[i], a.m.stride), a.m.ranges + (size_t)i * a.m.stride,
                     a.m.intensities + (size_t)i * a.m.stride};
  if (a.scan_sizes[i] == 0) return SlotBeams{0u, nullptr, nullptr};
  const uint32_t M = a.m.counts[i];
  const float* rg = reinterpret_cast<const float*>(a.scan_msgs + a.place[i]);
  return SlotBeams{M, rg, rg + M + 1};  // the intensities follow the ranges and their count
}

// a point (x, y, 0) in the target frame of a stream's rows xr {R_k0, R_k1, t_k, on}: p_target = R p + t, z = 0, so no
// R_k2 term, and no FMA (tests/scan_cloud_transform_oracle.py)
__device__ __forceinline__ void target_point(const float4 (&xr)[3], float x, float y, float (&X)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) X[k] = __fadd_rn(__fadd_rn(__fmul_rn(xr[k].x, x), __fmul_rn(xr[k].y, y)), xr[k].z);
}

}  // namespace
}  // namespace rpl
