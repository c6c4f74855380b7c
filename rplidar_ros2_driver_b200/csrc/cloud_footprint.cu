// cloud_footprint.cu -- the footprint pass of the PointCloud2 chain (DESIGN.md 5.7.1 "Footprints in the clouds"):
// between steps 1-3 (window, angle order, polar -> xyz) and step 4 (SOR) of oracle/cloud_oracle.cpp, every point a
// footprint polygon removes (oracle/scan_footprint_oracle.py, the rule of footprint_rule.cuh) is dropped from its
// scan's cloud.
//
// One CTA per scan over a persistent grid.  A scan with polygons stages them in shared memory (y negated for an
// inverted stream), tests every point of its row chunk by chunk, and compacts the kept points in place with a block
// scan: a chunk is read whole before any of it is written, and a point never moves forward, so the writes stay behind
// the reads and the angle order is kept.  Scans without polygons, or without points, are not touched.
#include <algorithm>
#include <cstddef>

#include "cloud_footprint_args.h"
#include "footprint_rule.cuh"
#include "rpl_device.cuh"

namespace rpl {
namespace {

constexpr int PT = 256;  // threads per CTA

__global__ void __launch_bounds__(PT) cloud_footprint_kernel(const __grid_constant__ CloudFootprintArgs a) {
  __shared__ ScanFootprint fp;
  __shared__ uint32_t s_warp[PT / 32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr uint32_t kY0 = offsetof(ScanFootprint, y) / 4, kY1 = offsetof(ScanFootprint, n_vertices) / 4;
  for (uint32_t s = blockIdx.x; s < a.n_scans; s += gridDim.x) {
    const ScanFootprint* src = a.footprints ? a.footprints + s / a.per : &a.one;
    const uint32_t np = src->n_polygons;
    if (np == 0) continue;
    const uint32_t m = a.point_counts[s];
    if (m == 0 || m > a.stride) continue;
    // the polygons, mirrored (y negated: exact) for an inverted stream
    const uint32_t flip = a.lidars && a.lidars[s / a.per].inverted ? 0x80000000u : 0u;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(src);
    uint32_t* d = reinterpret_cast<uint32_t*>(&fp);
    for (uint32_t k = tid; k < sizeof(ScanFootprint) / 4; k += PT) d[k] = w[k] ^ (k >= kY0 && k < kY1 ? flip : 0u);
    __syncthreads();
    float4* pts = a.xyzi + (size_t)s * a.stride;
    uint32_t done = 0;
    for (uint32_t c0 = 0; c0 < m; c0 += PT) {
      const uint32_t i = c0 + tid;
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
      uint32_t keep = 0;
      if (i < m) {
        p = pts[i];
        keep = footprint_removes(fp, np, [&](float* x, float* y) { *x = p.x, *y = p.y; }) ? 0u : 1u;
      }
      // exclusive block scan of keep; the chunk is read whole before the barrier, written after it
      const uint32_t inc = warp_inclusive_scan(keep);
      if (lane == 31) s_warp[warp] = inc;
      __syncthreads();
      uint32_t base = 0, tot = 0;
#pragma unroll
      for (int v = 0; v < PT / 32; ++v) {
        const uint32_t t = s_warp[v];
        if ((uint32_t)v < warp) base += t;
        tot += t;
      }
      __syncthreads();
      const uint32_t to = done + base + inc - keep;
      if (keep && to != i) pts[to] = p;
      done += tot;
    }
    if (tid == 0) a.point_counts[s] = done;
    __syncthreads();  // the next scan restages fp
  }
}

}  // namespace

cudaError_t launch_cloud_footprint(const CloudFootprintArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n_scans == 0) return cudaSuccess;
  // a persistent grid: as many CTAs as can be resident at once (the kernel's occupancy, asked once)
  static const int per_sm = [] {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, cloud_footprint_kernel, PT, 0);
    return std::max(n, 1);
  }();
  const int grid = (int)std::min<uint32_t>(a.n_scans, (uint32_t)(num_sms * per_sm));
  cloud_footprint_kernel<<<grid, PT, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rpl
