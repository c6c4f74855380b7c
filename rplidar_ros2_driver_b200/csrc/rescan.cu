// rescan.cu -- LaserScans re-gridded from the projected clouds (DESIGN.md 5.7.1 "LaserScans re-gridded from the
// projected clouds"), pointcloud_to_laserscan's cloudCallback, whose definition and CPU restatement is
// oracle/rescan_oracle.py: each point of a slot's projected cloud (the beams P keeps, through beam_point.cuh and the
// stream's transform rows: exactly the records scan_cloud_msgs publishes) inside the height band, the range window and
// the angular window lands in bin (int)((atan2(y, x) - angle_min) / angle_increment), which keeps the least range.
//
// One CTA per scan slot over a persistent grid.  The slot's grid lives in shared memory as float bits: every value is
// >= 0, so an integer atomicMin is the float min, and the result does not depend on the order of the points.  The grid
// is written straight into the slot's placed LaserScan message (msg_table_kernel sizes it from the stream's entry), or
// into its row.  No state is kept.
#include <algorithm>

#include "beam_point.cuh"
#include "msg_fixed.cuh"
#include "rescan_args.h"
#include "scan_cloud_point.cuh"

namespace rpl {
namespace {

constexpr int RT = 256;

__global__ void __launch_bounds__(RT) rescan_kernel(const __grid_constant__ RescanArgs a) {
  __shared__ uint32_t s_bins[kRescanMaxBins];
  const ScanCloudArgs& c = a.c;
  const uint32_t tid = threadIdx.x;
  for (uint32_t s = blockIdx.x; s < c.m.n; s += gridDim.x) {
    const uint32_t i = c.m.slot0 + s;
    if (c.m.out && c.m.sizes[i] == 0) continue;  // no message, or the messages do not fit
    const RescanGrid& g = a.grid ? a.grid[i / c.m.max_scans] : a.grid_one;
    for (uint32_t b = tid; b < g.bins; b += RT) s_bins[b] = g.seed;
    __syncthreads();
    const SlotBeams sb = slot_beams(c, i);
    const float inc = sb.M ? c.m.angle_increment[i] : 0.0f;
    float lo, cut;
    slot_window(c, i, &lo, &cut);
    float4 xr[3] = {};  // the stream's rows {R_k0, R_k1, t_k, on}; on 0: no transform
    if (c.transform) {
      const float4* rows = c.xf ? c.xf + 3 * (i / c.m.max_scans) : c.xf_one;
#pragma unroll
      for (int k = 0; k < 3; ++k) xr[k] = rows[k];
    }
    const double amin = g.angle_min, amax = g.angle_max, ainc = g.angle_increment;
    for (uint32_t j = tid; j < sb.M; j += RT) {
      const float r = sb.rg[j];
      if (!keep_beam(r, lo, cut)) continue;
      float x, y, p[3];
      beam_point(j, inc, r, &x, &y);
      if (xr[0].w != 0.0f) {
        target_point(xr, x, y, p);
      } else {
        p[0] = x;
        p[1] = y;
        p[2] = 0.0f;
      }
      if (p[2] > g.max_height || p[2] < g.min_height) continue;
      const double X = p[0], Y = p[1];
      // the products of floats are exact in double; the sum is rounded once and sqrt correctly
      const double range = __dsqrt_rn(__dadd_rn(__dmul_rn(X, X), __dmul_rn(Y, Y)));
      if (range < (double)g.range_min || range > (double)g.range_max) continue;
      const double angle = atan2_f64(Y, X);
      if (angle < amin || angle > amax) continue;
      const int index = __double2int_rz(__ddiv_rn(__dsub_rn(angle, amin), ainc));  // >= 0
      if (index >= (int)g.bins) continue;  // the package would write past its grid here
      atomicMin(&s_bins[index], __float_as_uint(__double2float_rn(range)));
    }
    __syncthreads();
    if (c.m.out) {
      const StreamMsgHeader& h = c.transform ? c.cloud_hdr[i / c.m.max_scans] : c.m.hdr[i / c.m.max_scans];
      uint8_t* msg = c.m.out + (c.m.offsets[i] - c.m.out_base);
      put_header<RT>(msg, h);
      uint8_t* body = msg + h.bytes;
      if (tid == 0) {
        uint32_t sec, nsec;
        msg_stamp(c.m.begin_us ? c.m.begin_us[i] : 0ull, c.m.clock_offset_ns, &sec, &nsec);
        put32(msg + 4, sec);
        put32(msg + 8, nsec);
        put32(body + 32 + 4 * g.bins, 0u);  // intensities: none
      }
      if (tid < 8) {  // angle_min, angle_max, angle_increment, time_increment 0, scan_time, range_min, range_max, ranges'
                      // count
        const float f = tid == 0 ? g.angle_min : tid == 1 ? g.angle_max : tid == 2 ? g.angle_increment
                        : tid == 4 ? g.scan_time : tid == 5 ? g.range_min : tid == 6 ? g.range_max : 0.0f;
        put32(body + 4 * tid, tid == 7 ? g.bins : __float_as_uint(f));
      }
      for (uint32_t b = tid; b < g.bins; b += RT) put32(body + 32 + 4 * b, s_bins[b]);
    } else {
      uint32_t* row = reinterpret_cast<uint32_t*>(a.out) + (size_t)i * g.bins;
      for (uint32_t b = tid; b < g.bins; b += RT) row[b] = s_bins[b];
    }
    __syncthreads();  // s_bins is seeded again for the next slot
  }
}

}  // namespace

cudaError_t launch_rescan(const RescanArgs& a, int num_sms, cudaStream_t stream) {
  if (a.c.m.n == 0) return cudaSuccess;
  static const int k = [] {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, rescan_kernel, RT, 0);
    return std::max(n, 1);
  }();
  rescan_kernel<<<(int)std::min<uint32_t>(a.c.m.n, (uint32_t)(num_sms * k)), RT, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rpl
