// scan_cloud.cu -- the projection of published LaserScans into PointCloud2 (DESIGN.md 5.7.1 "Clouds projected from the
// LaserScans"), laser_geometry's LaserProjection::projectLaser, whose definition and CPU restatement is
// oracle/scan_cloud_oracle.py: beam i is kept iff range_min <= r_i < cutoff, and becomes the record x, y, z = 0 and the
// chosen channels, the kept beams in beam order.  x, y is beam_point.cuh's point, the one the footprint stage of the
// filters tests.
//
// One CTA per scan slot over a persistent grid.  The count pass gives each slot's kept count, from which msg_table_kernel
// (cdr.cu) places a session's messages exactly; the write pass decides every beam again, compacts the kept ones chunk by
// chunk (a warp ballot for the lane's place, the warps' counts in shared memory for the block's) and writes each record
// straight into its row or into its message's data, and a message's fixed part from the stream's header and the call's
// tail.  Both passes read the ranges only once per beam; no state is kept.  A slot's beams are its row, or, in a push
// that returns both messages (push_scan_cloud_msgs), its LaserScan message where the push's scan kernels placed it.
// scan_cloud_kernel<true> moves each point into its stream's target frame (DESIGN.md 5.7.1 "Projected clouds in a target
// frame", tests/scan_cloud_transform_oracle.py) and may add the viewpoint; <false> is the projection without one.
#include <algorithm>

#include "beam_point.cuh"
#include "msg_fixed.cuh"
#include "scan_cloud_args.h"
#include "scan_cloud_point.cuh"

namespace rpl {
namespace {

constexpr int ST = 256;

__global__ void __launch_bounds__(ST) scan_cloud_count_kernel(const __grid_constant__ ScanCloudArgs a) {
  for (uint32_t s = blockIdx.x; s < a.m.n; s += gridDim.x) {
    const uint32_t i = a.m.slot0 + s;
    const SlotBeams sb = slot_beams(a, i);
    const uint32_t M = sb.M;
    const float* rg = sb.rg;
    float lo, cut;
    slot_window(a, i, &lo, &cut);
    uint32_t n = 0;
    for (uint32_t b0 = 0; b0 < M; b0 += ST) {
      const uint32_t j = b0 + threadIdx.x;
      n += __syncthreads_count(j < M && keep_beam(rg[j], lo, cut));
    }
    if (threadIdx.x == 0) a.kept[i] = n;
  }
}

// The message's header and tail: the LaserScan's and the channel set's, or a transforming call's (the target frame's,
// the tail with the viewpoint fields)
template <bool kXf>
__device__ __forceinline__ const StreamMsgHeader& cloud_header(const ScanCloudArgs& a, uint32_t i) {
  if constexpr (kXf) return a.cloud_hdr[i / a.m.max_scans];
  else return a.m.hdr[i / a.m.max_scans];
}
template <bool kXf>
__device__ __forceinline__ const auto& cloud_tail(const ScanCloudArgs& a) {
  if constexpr (kXf) return a.tail_xf;
  else return a.tail;
}

// 8 CTAs per SM: left to itself the compiler takes 40 registers for the two sources and the persistent grid loses a
// quarter of its CTAs, which costs the row path 8-10 %; at 32 nothing spills.  The transforming instantiation (kXf:
// each point moved into the target frame, DESIGN.md 5.7.1 "Projected clouds in a target frame") holds its stream's
// three rows besides: kXfBlocks CTAs per SM.
constexpr int kXfBlocks = 8;
template <bool kXf>
__global__ void __launch_bounds__(ST, kXf ? kXfBlocks : 8) scan_cloud_kernel(const __grid_constant__ ScanCloudArgs a) {
  __shared__ uint32_t s_warp[ST / 32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t words = a.point_step / 4, ch = a.channels;
  const auto& tail = cloud_tail<kXf>(a);
  for (uint32_t s = blockIdx.x; s < a.m.n; s += gridDim.x) {
    const uint32_t i = a.m.slot0 + s;
    const SlotBeams sb = slot_beams(a, i);
    const uint32_t M = sb.M;
    float ti;
    uint32_t* data;
    if (a.m.out) {
      if (a.m.sizes[i] == 0) continue;  // no message, or the messages do not fit
      const StreamMsgHeader& h = cloud_header<kXf>(a, i);
      uint8_t* msg = a.m.out + (a.m.offsets[i] - a.m.out_base);
      const uint32_t P = h.bytes + tail.bytes, n = a.kept[i];
      put_header<ST>(msg, h);
      for (uint32_t w = tid; w < tail.bytes / 4; w += ST) {
        const uint32_t v = w == tail.at_width ? n
                           : (w == tail.at_row_step || w == tail.at_data) ? a.point_step * n
                                                                          : tail.w[w];
        put32(msg + h.bytes + 4 * w, v);
      }
      const unsigned long long b = a.m.begin_us ? a.m.begin_us[i] : 0ull, e = a.m.end_us ? a.m.end_us[i] : 0ull;
      if (tid == 0) {
        uint32_t sec, nsec;
        msg_stamp(b, a.m.clock_offset_ns, &sec, &nsec);
        put32(msg + 4, sec);
        put32(msg + 8, nsec);
        msg[P + (size_t)a.point_step * n] = 1;  // is_dense: every kept point is finite
      }
      const bool mode_a = a.m.lidars ? a.m.lidars[i / a.m.max_scans].mode_a != 0 : a.m.mode_a != 0;
      ti = msg_time_increment(msg_period(b, e), mode_a, M);  // the LaserScan message's time_increment
      data = reinterpret_cast<uint32_t*>(msg + P);
    } else {
      ti = a.time_increment ? a.time_increment[i] : 0.0f;
      data = reinterpret_cast<uint32_t*>(a.points) + (size_t)s * a.m.stride * words;
    }
    const float *rg = sb.rg, *ig = sb.ig;
    const float inc = M ? a.m.angle_increment[i] : 0.0f;
    float lo, cut;
    slot_window(a, i, &lo, &cut);
    float4 xr[3];  // kXf: the stream's rows {R_k0, R_k1, t_k, on}
    if constexpr (kXf) {
      const float4* rows = a.xf ? a.xf + 3 * (i / a.m.max_scans) : a.xf_one;
#pragma unroll
      for (int k = 0; k < 3; ++k) xr[k] = rows[k];
    }
    uint32_t done = 0;
    for (uint32_t b0 = 0; b0 < M; b0 += ST) {
      const uint32_t j = b0 + tid;
      const float r = j < M ? rg[j] : 0.0f;
      const bool keep = j < M && keep_beam(r, lo, cut);
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, keep);
      if (lane == 0) s_warp[warp] = __popc(bal);
      __syncthreads();
      uint32_t base = 0, tot = 0;
#pragma unroll
      for (int v = 0; v < ST / 32; ++v) {
        const uint32_t t = s_warp[v];
        if ((uint32_t)v < warp) base += t;
        tot += t;
      }
      __syncthreads();  // s_warp is rewritten by the next chunk
      if (keep) {
        uint32_t* p = data + (size_t)(done + base + __popc(bal & ((1u << lane) - 1u))) * words;
        float x, y;
        beam_point(j, inc, r, &x, &y);
        if constexpr (kXf) {
          if (xr[0].w != 0.0f) {
            float X[3];
            target_point(xr, x, y, X);
            p[0] = __float_as_uint(X[0]);
            p[1] = __float_as_uint(X[1]);
            p[2] = __float_as_uint(X[2]);
          } else {
            p[0] = __float_as_uint(x);
            p[1] = __float_as_uint(y);
            p[2] = 0u;
          }
        } else {
          p[0] = __float_as_uint(x);
          p[1] = __float_as_uint(y);
          p[2] = 0u;
        }
        uint32_t k = 3;
        if (ch & kScanCloudIntensity) p[k++] = __float_as_uint(ig[j]);
        if (ch & kScanCloudIndex) p[k++] = j;
        if (ch & kScanCloudDistance) p[k++] = __float_as_uint(r);
        if (ch & kScanCloudTimestamp) p[k++] = __float_as_uint(__fmul_rn((float)j, ti));
        if constexpr (kXf) {
          if (ch & kScanCloudViewpoint) {  // the sensor origin in the target frame: t (a disabled entry's is 0)
            p[k] = __float_as_uint(xr[0].w != 0.0f ? xr[0].z : 0.0f);
            p[k + 1] = __float_as_uint(xr[0].w != 0.0f ? xr[1].z : 0.0f);
            p[k + 2] = __float_as_uint(xr[0].w != 0.0f ? xr[2].z : 0.0f);
          }
        }
      }
      done += tot;
    }
    if (!a.m.out && tid == 0) a.kept[i] = done;
  }
}

// a persistent grid: as many CTAs as can be resident at once (the kernel's occupancy, asked once)
template <class K>
int per_sm(K kernel) {
  int n = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, ST, 0);
  return std::max(n, 1);
}

}  // namespace

cudaError_t launch_scan_cloud_count(const ScanCloudArgs& a, int num_sms, cudaStream_t stream) {
  if (a.m.n == 0) return cudaSuccess;
  static const int k = per_sm(scan_cloud_count_kernel);
  scan_cloud_count_kernel<<<(int)std::min<uint32_t>(a.m.n, (uint32_t)(num_sms * k)), ST, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_scan_cloud(const ScanCloudArgs& a, int num_sms, cudaStream_t stream) {
  if (a.m.n == 0) return cudaSuccess;
  if (a.transform) {
    static const int k = per_sm(scan_cloud_kernel<true>);
    scan_cloud_kernel<true><<<(int)std::min<uint32_t>(a.m.n, (uint32_t)(num_sms * k)), ST, 0, stream>>>(a);
  } else {
    static const int k = per_sm(scan_cloud_kernel<false>);
    scan_cloud_kernel<false><<<(int)std::min<uint32_t>(a.m.n, (uint32_t)(num_sms * k)), ST, 0, stream>>>(a);
  }
  return cudaGetLastError();
}

}  // namespace rpl
