// msg_fixed.cuh -- the fixed parts a stream session's packed messages share (cdr.cu, scan_cloud.cu): the header words
// of a stream, the stamp of a scan on the caller's clock, and the LaserScan's timing members, so that a message built
// from a LaserScan carries that LaserScan's header and timing bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cdr_args.h"

namespace rpl {
namespace {

constexpr float kLaserScanRangeMin = 0.15f;  // the range_min every session LaserScan carries

__device__ __forceinline__ void put32(uint8_t* p, uint32_t v) { *reinterpret_cast<uint32_t*>(p) = v; }

// header.stamp of a scan-begin stamp b (SDK us) on the caller's clock: {0, 0} when unknown or not representable
__device__ __forceinline__ void msg_stamp(unsigned long long b, long long offset_ns, uint32_t* sec, uint32_t* nanosec) {
  *sec = 0;
  *nanosec = 0;
  if (b == 0) return;
  const long long t = (long long)(b * 1000ull + (unsigned long long)offset_ns);  // int64 ns, two's complement
  if (t < 0) return;
  const long long s = t / 1000000000ll;
  if (s > 2147483647ll) return;
  *sec = (uint32_t)s;
  *nanosec = (uint32_t)(t - s * 1000000000ll);
}

// rclcpp's Duration::seconds() of the stamp-to-stamp period (0 when either stamp is unknown or the period is not > 0)
__device__ __forceinline__ double msg_period(unsigned long long b, unsigned long long e) {
  if (b == 0 || e == 0 || e <= b) return 0.0;
  return (double)(long long)((e - b) * 1000ull) / 1e9;
}

// the LaserScan's time_increment of an n-beam scan over period d: d / n in Mode A, d / max(n - 1, 1) in Mode B
__device__ __forceinline__ float msg_time_increment(double d, bool mode_a, uint32_t n) {
  const double denom = mode_a ? (double)n : (double)(n > 1 ? n - 1 : 1);
  return __double2float_rn(d / denom);
}

// the header words of the stream's settings, stamp words left to the caller (no two threads write one word); T threads
template <int T>
__device__ __forceinline__ void put_header(uint8_t* msg, const StreamMsgHeader& h) {
  for (uint32_t w = threadIdx.x; w < h.bytes / 4; w += T)
    if (w != 1 && w != 2) put32(msg + 4 * w, h.w[w]);
}

}  // namespace
}  // namespace rpl
