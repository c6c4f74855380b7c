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

// fdlibm's atan and atan2 (s_atan.c, e_atan2.c), every double operation rounded as written (oracle/rescan_oracle.py
// atan_f64, atan2_f64): the angle of a point for the re-gridded scans (rescan.cu)
__constant__ double kAtanHi[4] = {4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01,
                                  1.57079632679489655800e+00};
__constant__ double kAtanLo[4] = {2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17,
                                  6.12323399573676603587e-17};
__constant__ double kAtanT[11] = {3.33333333333329318027e-01,  -1.99999999998764832476e-01, 1.42857142725034663711e-01,
                                  -1.11111104054623557880e-01, 9.09088713343650656196e-02,  -7.69187620504482999495e-02,
                                  6.66107313738753120669e-02,  -5.83357013379057348645e-02, 4.97687799461593236017e-02,
                                  -3.65315727442169155270e-02, 1.62858201153657823623e-02};
constexpr double kPiO4 = 7.8539816339744827900e-01, kPiO2 = 1.5707963267948965580e+00,
                 kPi = 3.1415926535897931160e+00, kPiLo = 1.2246467991473531772e-16, kAtanTiny = 1.0e-300;

__device__ __forceinline__ double atan_f64(double x) {
  const int hx = __double2hiint(x), ix = hx & 0x7fffffff;
  if (ix >= 0x44100000) {  // |x| >= 2^66, or NaN
    if (ix > 0x7ff00000 || (ix == 0x7ff00000 && __double2loint(x) != 0)) return __dadd_rn(x, x);
    return hx > 0 ? __dadd_rn(kAtanHi[3], kAtanLo[3]) : __dsub_rn(-kAtanHi[3], kAtanLo[3]);
  }
  int id;
  if (ix < 0x3fdc0000) {             // |x| < 0.4375
    if (ix < 0x3e200000) return x;   // |x| < 2^-29
    id = -1;
  } else {
    const double a = fabs(x);
    if (ix < 0x3ff30000) {           // |x| < 1.1875
      if (ix < 0x3fe60000) {         // 7/16 <= |x| < 11/16
        id = 0;
        x = __ddiv_rn(__dsub_rn(__dmul_rn(2.0, a), 1.0), __dadd_rn(2.0, a));
      } else {                       // 11/16 <= |x| < 19/16
        id = 1;
        x = __ddiv_rn(__dsub_rn(a, 1.0), __dadd_rn(a, 1.0));
      }
    } else if (ix < 0x40038000) {    // |x| < 2.4375
      id = 2;
      x = __ddiv_rn(__dsub_rn(a, 1.5), __dadd_rn(1.0, __dmul_rn(1.5, a)));
    } else {                         // 2.4375 <= |x| < 2^66
      id = 3;
      x = __ddiv_rn(-1.0, a);
    }
  }
  const double z = __dmul_rn(x, x), w = __dmul_rn(z, z);
  double s1 = kAtanT[10], s2 = kAtanT[9];
#pragma unroll
  for (int k = 8; k >= 0; k -= 2) s1 = __dadd_rn(kAtanT[k], __dmul_rn(w, s1));
#pragma unroll
  for (int k = 7; k >= 1; k -= 2) s2 = __dadd_rn(kAtanT[k], __dmul_rn(w, s2));
  s1 = __dmul_rn(z, s1);
  s2 = __dmul_rn(w, s2);
  const double xs = __dmul_rn(x, __dadd_rn(s1, s2));
  if (id < 0) return __dsub_rn(x, xs);
  const double r = __dsub_rn(kAtanHi[id], __dsub_rn(__dsub_rn(xs, kAtanLo[id]), x));
  return hx < 0 ? -r : r;
}

__device__ __forceinline__ double atan2_f64(double y, double x) {
  const int hx = __double2hiint(x), ix = hx & 0x7fffffff, hy = __double2hiint(y), iy = hy & 0x7fffffff;
  const unsigned lx = (unsigned)__double2loint(x), ly = (unsigned)__double2loint(y);
  if ((ix | ((lx | (0u - lx)) >> 31)) > 0x7ff00000u || (iy | ((ly | (0u - ly)) >> 31)) > 0x7ff00000u)
    return __dadd_rn(x, y);  // x or y is NaN
  if (((hx - 0x3ff00000) | (int)lx) == 0) return atan_f64(y);  // x = 1
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);           // 2 * sign(x) + sign(y)
  if ((iy | (int)ly) == 0) {                                    // y = 0
    if (m < 2) return y;
    return m == 2 ? __dadd_rn(kPi, kAtanTiny) : __dsub_rn(-kPi, kAtanTiny);
  }
  if ((ix | (int)lx) == 0) return hy < 0 ? __dsub_rn(-kPiO2, kAtanTiny) : __dadd_rn(kPiO2, kAtanTiny);  // x = 0
  if (ix == 0x7ff00000) {  // x = +-inf
    if (iy == 0x7ff00000) {
      const double q = m < 2 ? kPiO4 : __dmul_rn(3.0, kPiO4);
      return (m & 1) ? __dsub_rn(-q, kAtanTiny) : __dadd_rn(q, kAtanTiny);
    }
    if (m == 0) return 0.0;
    if (m == 1) return -0.0;
    return m == 2 ? __dadd_rn(kPi, kAtanTiny) : __dsub_rn(-kPi, kAtanTiny);
  }
  if (iy == 0x7ff00000) return hy < 0 ? __dsub_rn(-kPiO2, kAtanTiny) : __dadd_rn(kPiO2, kAtanTiny);  // y = +-inf
  const int k = (iy - ix) >> 20;
  double z;
  if (k > 60) z = __dadd_rn(kPiO2, __dmul_rn(0.5, kPiLo));  // |y / x| > 2^60
  else if (hx < 0 && k < -60) z = 0.0;                     // |y| / x < -2^60
  else z = atan_f64(fabs(__ddiv_rn(y, x)));
  switch (m) {
    case 0: return z;
    case 1: return -z;
    case 2: return __dsub_rn(kPi, __dsub_rn(z, kPiLo));
    default: return __dsub_rn(__dsub_rn(z, kPiLo), kPi);
  }
}

}  // namespace
}  // namespace rpl
