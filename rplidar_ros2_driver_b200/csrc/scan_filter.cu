// scan_filter.cu -- the LaserScan filter chain F(settings, scan) of DESIGN.md 5.7.1 "LaserScan filters", whose
// definition and CPU restatement is oracle/scan_filter_oracle.py: angular mask, range window, intensity floor, speckle
// and veiling-point removal, in place on published LaserScans.
//
// One CTA per scan over a persistent grid.  The scan's ranges are staged in shared memory with the three per-beam
// stages applied on the way in; the speckle and veiling stages each decide every beam from the staged ranges into a
// bitmap (one ballot word per warp), then mark the removed beams NaN; the ranges go back at the end.  A scan's
// (sin, cos) table of k * angle_increment, k <= 16, comes from a double polynomial with every operation rounded as
// written, so that the decisions are the restatement's bit for bit.  The footprint stage
// (oracle/scan_footprint_oracle.py) runs beside the three per-beam stages: a scan with polygons stages them in shared
// memory, and every beam still finite after the other per-beam stages takes its point from the same double polynomial
// and is tested against each polygon.
#include <algorithm>

#include "beam_point.cuh"
#include "footprint_rule.cuh"
#include "scan_args.h"
#include "scan_filter_args.h"

namespace rpl {
namespace {

constexpr int FT = 256;
constexpr uint32_t kNanBits = 0x7FC00000u;

struct FilterSmem {
  float r[kScanFilterMaxBeams];
  uint32_t removed[kScanFilterMaxBeams / 32];
  float sk[kScanFilterMaxWindow + 1], ck[kScanFilterMaxWindow + 1];
  ScanFootprint fp;
};

// the footprint stage: the point of beam i at range r (finite) is inside a polygon whose invert is 0, or outside one
// whose invert is 1 (footprint_rule.cuh)
__device__ __forceinline__ bool footprint(const ScanFootprint& fp, uint32_t np, uint32_t i, float r, float inc) {
  return footprint_removes(fp, np, [&](float* x, float* y) { beam_point(i, inc, r, x, y); });
}

// speckle: a finite beam with fewer than n neighbours within w beams and max_diff of its range
__device__ __forceinline__ bool speckle(const float* r, uint32_t i, uint32_t M, uint32_t w, uint32_t n, float max_diff) {
  const float v = r[i];
  if (!isfinite(v)) return false;
  uint32_t cnt = 0;
  for (uint32_t d = 1; d <= w; ++d) {
    if (i >= d) {
      const float u = r[i - d];
      cnt += isfinite(u) && fabsf(__fsub_rn(u, v)) <= max_diff;
    }
    if (i + d < M) {
      const float u = r[i + d];
      cnt += isfinite(u) && fabsf(__fsub_rn(u, v)) <= max_diff;
    }
  }
  return cnt < n;
}

// veiling: beam j is the far end of a pair whose segment is within the shadow angle of the near beam's line of sight
__device__ __forceinline__ bool veiling(const FilterSmem& sm, uint32_t j, uint32_t M, uint32_t w, float tan_shadow) {
  const float rj = sm.r[j];
  if (!(isfinite(rj) && rj > 0.0f)) return false;
  for (uint32_t k = 1; k <= w; ++k) {
    const float xk = __fmul_rn(rj, sm.ck[k]), yk = __fmul_rn(rj, sm.sk[k]);
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      if (side == 0 ? j < k : j + k >= M) continue;
      const float ri = sm.r[side == 0 ? j - k : j + k];
      if (!(isfinite(ri) && ri > 0.0f && ri < rj)) continue;
      const float dx = __fsub_rn(xk, ri);
      if (dx > 0.0f && yk < __fmul_rn(tan_shadow, dx)) return true;
    }
  }
  return false;
}

// one stage's decisions into sm.removed (every warp runs the same trip count: the ballot needs the whole warp)
template <class Decide>
__device__ __forceinline__ void decide(FilterSmem& sm, uint32_t M, Decide fn) {
  for (uint32_t base = 0; base < M; base += FT) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, i < M && fn(i));
    if ((threadIdx.x & 31u) == 0) sm.removed[i >> 5] = b;
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < M; i += FT)
    if ((sm.removed[i >> 5] >> (i & 31u)) & 1u) sm.r[i] = __uint_as_float(kNanBits);
  __syncthreads();
}

// a grid constant: `one_footprint` is read in place in the parameter space by address, without a local copy
__global__ void __launch_bounds__(FT) scan_filter_kernel(const __grid_constant__ ScanFilterArgs a) {
  __shared__ FilterSmem sm;
  for (uint32_t s = blockIdx.x; s < a.n_scans; s += gridDim.x) {
    const ScanFilter& f = a.filters ? a.filters[s / a.per_filter] : a.one;
    if (!f.enabled) continue;
    const uint32_t M = min(a.beam_counts[s], kScanFilterMaxBeams);
    if (M == 0) continue;
    float* rg;
    const float* ig;
    if (a.msg_out) {
      const unsigned long long pl = a.place[s];
      if (pl & kOutSkip) continue;
      rg = reinterpret_cast<float*>(a.msg_out + pl);
      ig = rg + M + 1;
    } else {
      rg = a.ranges + (size_t)s * a.stride;
      ig = a.intensities + (size_t)s * a.stride;
    }
    const float inc = a.angle_increment[s];
    const uint32_t sw = f.speckle_window, hw = f.shadow_window;
    if (threadIdx.x >= 1 && threadIdx.x <= hw) {
      double sn, cs;
      sincos_f64(__dmul_rn((double)threadIdx.x, (double)inc), &sn, &cs);
      sm.sk[threadIdx.x] = __double2float_rn(sn);
      sm.ck[threadIdx.x] = __double2float_rn(cs);
    }
    const ScanFootprint* fp = a.footprints ? a.footprints + s / a.per_filter : &a.one_footprint;
    const uint32_t np = fp->n_polygons;
    if (np) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(fp);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.fp);
      for (uint32_t w = threadIdx.x; w < sizeof(ScanFootprint) / 4; w += FT) dst[w] = src[w];
      __syncthreads();
    }
    // stages 1-3 and the footprint: angular mask, range window, intensity floor, polygons
    for (uint32_t i = threadIdx.x; i < M; i += FT) {
      float v = rg[i];
      if (isfinite(v)) {
        const float ang = __fmul_rn((float)i, inc);
        bool rm = v < f.range_lo || v > f.range_hi || ig[i] < f.intensity_min;
#pragma unroll
        for (int k = 0; k < 4; ++k) rm = rm || (f.mask_lo[k] <= ang && ang <= f.mask_hi[k]);
        rm = rm || (np && footprint(sm.fp, np, i, v, inc));
        if (rm) v = __uint_as_float(kNanBits);
      }
      sm.r[i] = v;
    }
    __syncthreads();
    if (sw > 0) {
      const uint32_t n = f.speckle_min_neighbours;
      const float d = f.speckle_max_diff;
      decide(sm, M, [&](uint32_t i) { return speckle(sm.r, i, M, sw, n, d); });
    }
    if (hw > 0) {
      const float t = f.shadow_tan;
      decide(sm, M, [&](uint32_t j) { return veiling(sm, j, M, hw, t); });
    }
    for (uint32_t i = threadIdx.x; i < M; i += FT) rg[i] = sm.r[i];
    __syncthreads();  // the next scan restages sm
  }
}

}  // namespace

cudaError_t launch_scan_filter(const ScanFilterArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n_scans == 0) return cudaSuccess;
  const int grid = (int)std::min<uint32_t>(a.n_scans, (uint32_t)num_sms * 4u);
  scan_filter_kernel<<<grid, FT, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rpl
