// beam_point.cuh -- the point of a LaserScan beam, shared by the footprint stage of the filters (scan_filter.cu) and
// the scan projection (scan_cloud.cu), so that a projected point is exactly the point the footprint stage tested.
// (sin, cos) of i * angle_increment come from a double polynomial with every operation rounded as written
// (oracle/scan_filter_oracle.py sincos_f64); the point is (fl(r * c), fl(r * s)) with (s, c) rounded to float once
// (oracle/scan_footprint_oracle.py beam_points).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {
namespace {

// Cody-Waite split of pi/2 and fdlibm's kernel polynomials (oracle/scan_filter_oracle.py sincos_f64)
constexpr double kTwoOverPi = 6.36619772367581382433e-01;
constexpr double kPio2_1 = 1.57079632673412561417e+00;
constexpr double kPio2_1t = 6.07710050650619224932e-11;
__constant__ double kSinC[6] = {-1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04,
                                2.75573137070700676789e-06, -2.50507602534068634195e-08, 1.58969099521155010221e-10};
__constant__ double kCosC[6] = {4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05,
                                -2.75573143513906633035e-07, 2.08757232129817482790e-09, -1.13596475577881948265e-11};

__device__ __forceinline__ void sincos_f64(double x, double* sn, double* cs) {
  const double q = rint(__dmul_rn(x, kTwoOverPi));
  const double r = __dsub_rn(__dsub_rn(x, __dmul_rn(q, kPio2_1)), __dmul_rn(q, kPio2_1t));
  const double z = __dmul_rn(r, r);
  double ps = kSinC[5], pc = kCosC[5];
#pragma unroll
  for (int i = 4; i >= 0; --i) {
    ps = __dadd_rn(kSinC[i], __dmul_rn(z, ps));
    pc = __dadd_rn(kCosC[i], __dmul_rn(z, pc));
  }
  const double s = __dadd_rn(r, __dmul_rn(__dmul_rn(r, z), ps));
  const double c = __dadd_rn(__dsub_rn(1.0, __dmul_rn(0.5, z)), __dmul_rn(__dmul_rn(z, z), pc));
  switch ((int)q & 3) {
    case 0: *sn = s; *cs = c; break;
    case 1: *sn = c; *cs = -s; break;
    case 2: *sn = -s; *cs = -c; break;
    default: *sn = -c; *cs = s; break;
  }
}

// the point of beam i at range r: i * inc is exact in double (i < 2^13, inc a float)
__device__ __forceinline__ void beam_point(uint32_t i, float inc, float r, float* x, float* y) {
  double sn, cs;
  sincos_f64(__dmul_rn((double)i, (double)inc), &sn, &cs);
  *x = __fmul_rn(r, __double2float_rn(cs));
  *y = __fmul_rn(r, __double2float_rn(sn));
}

}  // namespace
}  // namespace rpl
