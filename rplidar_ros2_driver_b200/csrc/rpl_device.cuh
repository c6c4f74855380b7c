// rpl_device.cuh -- device-side building blocks shared by the scan kernels.
//
// Everything here reproduces the reference's scalar arithmetic bit for bit; every float
// operation is an explicit round-to-nearest intrinsic (no FMA contraction: the x86-64
// reference build rounds the multiply and the add separately, SURVEY.md 7) and the library
// is compiled without --use_fast_math.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {

constexpr uint32_t kKeySpace = 65536;  // angle_z_q14 is a u16: 65536 units = 360 degrees
constexpr uint32_t kResultOk = 0u;
constexpr uint32_t kResultInvalidData = 0x80008000u;    // SL_RESULT_INVALID_DATA
constexpr uint32_t kResultOperationFail = 0x80008001u;  // SL_RESULT_OPERATION_FAIL

// A packed node (reference sl_lidar_cmd.h:272-278) seen as two little-endian words:
//   x = angle_z_q14 | dist_mm_q2[15:0] << 16
//   y = dist_mm_q2[31:16] | quality << 16 | flag << 24
// dist_mm_q2 sits at the unaligned byte offset 2, so it is never dereferenced directly.
__device__ __forceinline__ uint32_t node_key(uint2 n) { return n.x & 0xFFFFu; }
__device__ __forceinline__ uint32_t node_dist(uint2 n) { return __funnelshift_r(n.x, n.y, 16); }
__device__ __forceinline__ uint32_t node_quality(uint2 n) { return (n.y >> 16) & 0xFFu; }
__device__ __forceinline__ uint2 node_with_key(uint2 n, uint32_t key) {
  n.x = (n.x & 0xFFFF0000u) | (key & 0xFFFFu);
  return n;
}

// getAngle(hq): angle_z_q14 * 90.f / 16384.f (reference sl_lidar_driver.cpp:102-105).
// Both operations are exact (key*90 < 2^24, then a power-of-two scale).
__device__ __forceinline__ float key_to_deg(uint32_t key) {
  return __fmul_rn(__fmul_rn(__uint2float_rn(key), 90.0f), 1.0f / 16384.0f);
}
// setAngle(hq, v): angle_z_q14 = (u16)(u32)(v * 16384.f / 90.f) (reference :107-110).
// The division by 90 is one multiply + two FMAs (Markstein's reciprocal refinement, as in dist_to_m below) for
// every angle this path can produce (0 <= deg <= 720): oracle/check_div90.c proves the quotient bit-identical to
// the IEEE one for EVERY float in [0, 1024], denormals included.  Anything else takes the division itself.
__device__ __forceinline__ uint32_t deg_to_key(float deg) {
  const float x = __fmul_rn(deg, 16384.0f);
  float q;
  if (deg >= 0.0f && deg <= 1024.0f) {
    const float r = 1.0f / 90.0f;  // RN(1/90) = 0x1.6c16c2p-7
    const float q0 = __fmul_rn(x, r);
    const float e = __fmaf_rn(-q0, 90.0f, x);
    q = __fmaf_rn(e, r, q0);
  } else {
    q = __fdiv_rn(x, 90.0f);
  }
  return __float2uint_rz(q) & 0xFFFFu;
}
// inc_origin_angle = 360.f / count (reference :130)
__device__ __forceinline__ float ascend_step(uint32_t count) {
  return __fdiv_rn(360.0f, __uint2float_rn(count));
}
// fill of an unmeasured node i >= 1 (reference :171-178)
__device__ __forceinline__ uint32_t ascend_fill_key(float front_deg, uint32_t i, float step) {
  float a = __fadd_rn(front_deg, __fmul_rn(__uint2float_rn(i), step));
  if (a > 360.0f) a = __fsub_rn(a, 360.0f);
  return deg_to_key(a);
}
// head tune (reference :133-147): walk back from the first measured node, re-quantising at
// every step.  Only node 0's value survives (the fill overwrites the others), but it depends
// on the whole chain, so it is reproduced serially.  Once the chain clamps to 0 it stays 0.
__device__ __forceinline__ uint32_t ascend_head_key(uint32_t first_key, uint32_t first_index,
                                                    float step) {
  uint32_t k = first_key;
  for (uint32_t j = first_index; j > 0 && k != 0; --j) {
    float a = __fsub_rn(key_to_deg(k), step);
    if (a < 0.0f) a = 0.0f;
    k = deg_to_key(a);
  }
  return k;
}

// publish_scan unpack (reference rplidar_node.cpp:586-590)
__device__ __forceinline__ float key_to_rad(uint32_t key) {
  // float angle_rad = angle_deg * (M_PI / 180.0f): double product rounded to float
  const double kDegToRad = 3.14159265358979323846 / 180.0;
  return __double2float_rn(__dmul_rn((double)key_to_deg(key), kDegToRad));
}
// dist_m = dist_mm_q2 / 4000.0f, correctly rounded.  One multiply + two FMAs (Markstein's
// reciprocal refinement) instead of the generic division sequence; proven bit-identical to
// the IEEE quotient for every float a u32 converts to by oracle/check_div4000.c.
__device__ __forceinline__ float dist_to_m(uint32_t dist_q2) {
  const float x = __uint2float_rn(dist_q2);
  const float r = 1.0f / 4000.0f;  // RN(1/4000) = 0x1.0624dep-12
  const float q0 = __fmul_rn(x, r);
  const float e = __fmaf_rn(-q0, 4000.0f, x);
  return __fmaf_rn(e, r, q0);
}
// (float)q for q < 2^23 without the conversion pipe: 2^23 + q is exact, minus 2^23 is exact
__device__ __forceinline__ float small_uint_to_float(uint32_t q) {
  return __fsub_rn(__uint_as_float(0x4B000000u | q), 8388608.0f);
}
__device__ __forceinline__ float quality_to_intensity(uint32_t q, bool new_protocol) {
  return small_uint_to_float(new_protocol ? q : (q >> 2));
}
// the same intensity taken straight from node word y, with the protocol's shift and mask fixed once per launch
struct IntensityOf {
  uint32_t shift, mask;
  __device__ __forceinline__ explicit IntensityOf(bool new_protocol)
      : shift(new_protocol ? 16u : 18u), mask(new_protocol ? 0xFFu : 0x3Fu) {}
  __device__ __forceinline__ uint32_t units(uint32_t y) const { return (y >> shift) & mask; }
  __device__ __forceinline__ float operator()(uint32_t y) const { return small_uint_to_float(units(y)); }
};

// LaserScan.angle_increment (reference rplidar_node.cpp:633-634 Mode A, :664-666 Mode B)
__device__ __forceinline__ float angle_increment(uint32_t m, bool mode_a) {
  const double kTwoPi = 2.0 * 3.14159265358979323846;
  const uint32_t d = mode_a ? m : (m > 1 ? m - 1 : 1);
  return __double2float_rn(__ddiv_rn(kTwoPi, (double)d));
}
// Mode A bin of a measured point (reference rplidar_node.cpp:641-652); always < m for m >= 1
// because angle_rad <= 6.28308964 < 2*pi, but the reference's bounds check is kept by callers.
__device__ __forceinline__ int mode_a_bin(uint32_t key, float inc, bool inverted) {
  const double kTwoPi = 2.0 * 3.14159265358979323846;
  float a = key_to_rad(key);
  if (inverted) {
    a = __double2float_rn(__dsub_rn(kTwoPi, (double)a));
    if ((double)a >= kTwoPi) a = __double2float_rn(__dsub_rn((double)a, kTwoPi));
  }
  return __float2int_rz(__fdiv_rn(__fsub_rn(a, 0.0f), inc));
}

// Mode A bin without floating point for almost all keys.  The reference's float chain computes
// (k * 2pi/65536) / (2pi/M) with three float roundings (angle_rad, angle_increment, the
// quotient; the double-precision steps add < 1e-14): relative error <= 3 * 2^-24 of a quotient
// < M, i.e. at most 3M * 2^-24 bins (4M * 2^-24 for inverted scans, where 2pi - angle adds an
// absolute 2^-24 * 2pi).  In units of 2^-16 bin that is M/64, so whenever the exact ratio
// k*M/65536 (resp. (65536-k)*M/65536) has a fractional part further than g = M/32 + 2 units (twice
// the bound) from both bin edges, truncation of the float result equals the integer quotient; only
// the keys closer than that (a share M / 2^20 of them: 0.3 % for a 3200-beam scan, 6 % at 65536) and
// key 0 of inverted scans (the reference wraps it to 1.7e-7) take the exact chain.
// tests/test_device_math_proofs.py checks the claim against the float chain for every key over
// thousands of beam counts.
__device__ __forceinline__ int mode_a_bin_fast(uint32_t key, uint32_t m, float inc, bool inverted) {
  const uint32_t kk = inverted ? (65536u - key) : key;
  const uint32_t t = kk * m;  // < 2^32: kk <= 65535 on this branch, m <= 65536
  const uint32_t frac = t & 0xFFFFu;
  const uint32_t g = (m >> 5) + 2u;
  if ((!inverted || key != 0u) && (frac - g) <= (65536u - 2u * g)) return (int)(t >> 16);
  return mode_a_bin(key, inc, inverted);
}

// ---- counter-based splitmix64 (same definition as oracle/scan_oracle.cpp) --------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ---- small block-level helpers -----------------------------------------------------------
__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ uint32_t warp_min(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= (uint32_t)o) v += t;
  }
  return v;
}

// L2 residency control.  A scan tile is read twice (mark pass, place pass): the first read
// asks L2 to keep the lines (evict_last), the second read and all output stores mark their
// lines evict_first so that the 1 GB/launch output stream does not push tiles out of the
// 50 MB L2 before their second read.  The two-CTA cluster kernel reads each node once and marks
// its loads and stores evict_normal, which it measured faster than evict_first (scan_tma.cu).
// The policies are the fixed encodings createpolicy.fractional.L2::evict_{last,first,normal} (1.0)
// produces (the same constants CUTLASS passes as TMA cache hints); as immediates they live in
// uniform registers instead of being re-broadcast from a per-thread register at every access.
__device__ __forceinline__ uint64_t l2_policy_evict_last() { return 0x14F0000000000000ull; }
__device__ __forceinline__ uint64_t l2_policy_evict_first() { return 0x12F0000000000000ull; }
__device__ __forceinline__ uint64_t l2_policy_evict_normal() { return 0x1000000000000000ull; }
__device__ __forceinline__ uint4 ld_hint_v4(const void* p, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint2 ld_hint_v2(const void* p, uint64_t pol) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;"
               : "=r"(r.x), "=r"(r.y)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void st_hint_v2(uint2* p, uint2 v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol));
}

__device__ __forceinline__ void st_f32x4_if(float4* p, float4 v, uint64_t pol, uint32_t pred) {
  asm volatile(
      "{ .reg .pred q; setp.ne.u32 q, %6, 0;\n\t"
      "@q st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5; }" ::"l"(p),
      "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol), "r"(pred));
}
// PointCloud2 window test (oracle/cloud_oracle.cpp step 1); NaN-free inputs
__device__ __forceinline__ bool cloud_keep(float dm, float inten, float rmin, float rmax, float imin) {
  return !(dm < rmin) && !(dm > rmax) && !(inten < imin);
}

// streaming global load: inputs are read at most twice
__device__ __forceinline__ uint2 ld_stream_v2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

}  // namespace rpl
