// footprint_rule.cuh -- the footprint decision of oracle/scan_footprint_oracle.py, shared by the LaserScan filter
// (scan_filter.cu) and the PointCloud2 footprint pass (cloud_footprint.cu), so that both outputs apply one rule.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "scan_filter_args.h"

namespace rpl {

// the point point(&x, &y) gives is removed when it is inside one of the first np polygons of fp whose invert is 0, or
// outside one whose invert is 1: the crossing-number rule, every float operation rounded as written.  The caller forms
// the point inside the rule (a functor, not two arguments) so that the compiler sees one expression per decision
// whoever calls it.
template <class Point>
__device__ __forceinline__ bool footprint_removes(const ScanFootprint& fp, uint32_t np, Point point) {
  float x, y;
  point(&x, &y);
  for (uint32_t p = 0; p < np; ++p) {
    const uint32_t n = fp.n_vertices[p];
    float xa = fp.x[p][n - 1], ya = fp.y[p][n - 1];
    bool in = false;
    for (uint32_t k = 0; k < n; ++k) {
      const float xb = fp.x[p][k], yb = fp.y[p][k];
      if ((ya > y) != (yb > y) &&
          x < __fadd_rn(xa, __fdiv_rn(__fmul_rn(__fsub_rn(xb, xa), __fsub_rn(y, ya)), __fsub_rn(yb, ya))))
        in = !in;
      xa = xb;
      ya = yb;
    }
    if (in != (fp.invert[p] != 0)) return true;
  }
  return false;
}

}  // namespace rpl
