// cdr.cu -- LaserScan / PointCloud2 -> wire (SURVEY.md 8(f) rank 3: the step AFTER the hot path).
//
// The reference hands a sensor_msgs::msg::LaserScan to rclcpp (src/rplidar_node.cpp:679) and the RMW
// layer serialises it to CDR before it reaches the wire.  Here the serialised message is produced on the
// device, straight from the scan kernels' outputs, so that the host can publish the bytes as they are
// (rclcpp::SerializedMessage, INTEGRATION.md 4c) without building the message or copying the arrays
// again.  Encoding: XCDR version 1, little endian, the representation ROS 2's RMW implementations put
// on the wire -- 4-byte encapsulation header {0x00,0x01,0x00,0x00}, then the members in declaration
// order, every primitive aligned to its size relative to the first byte after that header, strings as
// uint32 length (terminating NUL included) + bytes, sequences as uint32 count + elements.
//   sensor_msgs/LaserScan:   header{stamp{int32 sec, uint32 nanosec}, string frame_id}, 7 x float32,
//                            float32[] ranges, float32[] intensities
//   sensor_msgs/PointCloud2: header, uint32 height, width, PointField[] fields{string name, uint32
//                            offset, uint8 datatype, uint32 count}, bool is_bigendian, uint32
//                            point_step, row_step, uint8[] data, bool is_dense
// The fixed part of each message (everything but the arrays) is a host-built template with a handful
// of 4-byte fields patched per message; the arrays are copied coalesced.
// PARITY UNPINNED: the reference holds no serialiser (it lives in the RMW dependency); the format
// follows the OMG CDR rules above and oracle/cdr_oracle.py restates it independently in numpy.
#include "cdr_args.h"
#include "rpl_device.cuh"
#include "scan_args.h"

namespace rpl {

namespace {

constexpr int CT = 256;

__device__ __forceinline__ void put32(uint8_t* p, uint32_t v) { *reinterpret_cast<uint32_t*>(p) = v; }

__global__ void __launch_bounds__(CT) laserscan_cdr_kernel(LaserScanCdrArgs a, CdrTemplate t) {
  const uint32_t s = blockIdx.y;
  const uint32_t n = a.beam_counts[s];
  uint8_t* msg = a.cdr_out + (size_t)s * a.cdr_stride;
  const uint32_t P = t.prefix_bytes;  // multiple of 4; ends with the ranges count
  if (blockIdx.x == 0) {
    for (uint32_t w = threadIdx.x; w < P / 4; w += CT) put32(msg + 4 * w, reinterpret_cast<const uint32_t*>(t.prefix)[w]);
    __syncthreads();
    if (threadIdx.x == 0) {
      const LaserScanMeta m = a.meta[s];
      put32(msg + 4, (uint32_t)m.stamp_sec);
      put32(msg + 8, m.stamp_nanosec);
      uint8_t* f = msg + P - 32;  // 7 floats, then the ranges count
      put32(f + 0, __float_as_uint(m.angle_min));
      put32(f + 4, __float_as_uint(m.angle_max));
      put32(f + 8, __float_as_uint(a.angle_increment ? a.angle_increment[s] : m.angle_increment));
      put32(f + 12, __float_as_uint(m.time_increment));
      put32(f + 16, __float_as_uint(m.scan_time));
      put32(f + 20, __float_as_uint(m.range_min));
      put32(f + 24, __float_as_uint(m.range_max));
      put32(f + 28, n);
      put32(msg + P + 4 * (size_t)n, n);  // intensities count
      if (a.cdr_sizes) a.cdr_sizes[s] = P + 8 * n + 4;
    }
  }
  uint32_t* r_out = reinterpret_cast<uint32_t*>(msg + P);
  uint32_t* i_out = r_out + n + 1;
  const uint32_t* r_in = reinterpret_cast<const uint32_t*>(a.ranges + (size_t)s * a.stride);
  const uint32_t* i_in = reinterpret_cast<const uint32_t*>(a.intensities + (size_t)s * a.stride);
  for (uint32_t i = blockIdx.x * CT + threadIdx.x; i < n; i += gridDim.x * CT) {
    r_out[i] = __ldg(r_in + i);
    i_out[i] = __ldg(i_in + i);
  }
}

__global__ void __launch_bounds__(CT) pointcloud2_cdr_kernel(PointCloudCdrArgs a, CdrTemplate t) {
  const uint32_t s = blockIdx.y;
  const uint32_t n = a.point_counts[s];
  uint8_t* msg = a.cdr_out + (size_t)s * a.cdr_stride;
  const uint32_t P = t.prefix_bytes;  // multiple of 4; ends with the data length
  if (blockIdx.x == 0) {
    for (uint32_t w = threadIdx.x; w < P / 4; w += CT) put32(msg + 4 * w, reinterpret_cast<const uint32_t*>(t.prefix)[w]);
    __syncthreads();
    if (threadIdx.x == 0) {
      put32(msg + 4, (uint32_t)a.stamps[2 * s]);
      put32(msg + 8, a.stamps[2 * s + 1]);
      put32(msg + t.patch_width, n);         // width (height = 1: unorganised cloud)
      put32(msg + t.patch_row_step, 16u * n);
      put32(msg + P - 4, 16u * n);           // data length
      msg[P + 16 * (size_t)n] = 1;           // is_dense: the cloud path drops unmeasured points
      if (a.cdr_sizes) a.cdr_sizes[s] = P + 16 * n + 1;
    }
  }
  // the prefix length follows from the frame id: 16-byte stores only when it happens to be a multiple of 16
  uint4* d_out = reinterpret_cast<uint4*>(msg + P);
  const uint4* d_in = reinterpret_cast<const uint4*>(a.xyzi + (size_t)s * a.stride * 4);
  if ((P & 15u) == 0) {
    for (uint32_t i = blockIdx.x * CT + threadIdx.x; i < n; i += gridDim.x * CT) d_out[i] = __ldg(d_in + i);
  } else {
    uint32_t* o = reinterpret_cast<uint32_t*>(msg + P);
    const uint32_t* in = reinterpret_cast<const uint32_t*>(d_in);
    for (uint32_t i = blockIdx.x * CT + threadIdx.x; i < 4 * n; i += gridDim.x * CT) o[i] = __ldg(in + i);
  }
}

// ---- packed messages of a stream session's push -----------------------------------------------------------------
constexpr int MT = 1024;  // the sizes and offsets pass: one CTA

__device__ __forceinline__ uint32_t msg_bytes(MsgKind kind, uint32_t header_bytes, uint32_t n) {
  return kind == MsgKind::kLaserScan ? header_bytes + 32 + 8 * n + 4 : header_bytes + 116 + 16 * n + 1;
}

// One CTA, the slots in tiles of MT: sizes, the exclusive scan of the sizes rounded up to 16 (the carry passes from
// tile to tile), the end of the last message; then every size again, or 0 when the messages do not fit.
__global__ void __launch_bounds__(MT) msg_table_kernel(MsgTableArgs a) {
  __shared__ unsigned long long s_warp[MT / 32];
  __shared__ unsigned long long s_end;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_end = 0;
  unsigned long long carry = 0;
  auto size_of = [&](uint32_t i) -> uint32_t {
    const uint32_t n = a.counts[i];
    const bool has = a.kind == MsgKind::kLaserScan
                         ? n > 0
                         : a.views[i].y > 0 && !(a.clouds && a.clouds[i / a.max_scans].route == kCloudOff);
    return has ? msg_bytes(a.kind, a.hdr[i / a.max_scans].bytes, n) : 0u;
  };
  for (uint32_t t0 = 0; t0 < a.n_slots; t0 += MT) {
    const uint32_t i = t0 + tid;
    const uint32_t sz = i < a.n_slots ? size_of(i) : 0u;
    const unsigned long long v = (sz + 15u) & ~15u;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= (uint32_t)o) inc += u;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long base = 0, tile = 0;
    for (uint32_t w = 0; w < MT / 32; ++w) {
      const unsigned long long x = s_warp[w];
      if (w < warp) base += x;
      tile += x;
    }
    const unsigned long long off = carry + base + inc - v;
    if (i < a.n_slots) {
      a.offsets[i] = off;
      if (sz) atomicMax(&s_end, off + sz);
    }
    carry += tile;
    __syncthreads();  // s_warp is rewritten by the next tile
  }
  const unsigned long long total = s_end;
  const bool fits = total <= a.capacity;
  for (uint32_t i = tid; i < a.n_slots; i += MT) a.sizes[i] = fits ? size_of(i) : 0u;
  if (tid == 0) *a.total = total;
}

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

// the header words of the stream's settings, stamp words left to the caller (no two threads write one word); T threads
template <int T = CT>
__device__ __forceinline__ void put_header(uint8_t* msg, const StreamMsgHeader& h) {
  for (uint32_t w = threadIdx.x; w < h.bytes / 4; w += T)
    if (w != 1 && w != 2) put32(msg + 4 * w, h.w[w]);
}

// LaserScan message i's fixed part -- header, stamp, the 7 floats, both sequence lengths -- for n beams, by the T threads
// of a CTA; P = h.bytes + 32, where the ranges start
template <int T>
__device__ __forceinline__ void put_laserscan_fixed(const MsgWriteArgs& a, uint32_t i, uint32_t n, const StreamMsgHeader& h,
                                                    uint32_t P, uint8_t* msg) {
  put_header<T>(msg, h);
  if (threadIdx.x == 0) {
    const unsigned long long b = a.begin_us ? a.begin_us[i] : 0ull, e = a.end_us ? a.end_us[i] : 0ull;
    uint32_t sec, nsec;
    msg_stamp(b, a.clock_offset_ns, &sec, &nsec);
    const double d = msg_period(b, e);
    const bool mode_a = a.lidars ? a.lidars[i / a.max_scans].mode_a != 0 : a.mode_a != 0;
    const double denom = mode_a ? (double)n : (double)(n > 1 ? n - 1 : 1);
    put32(msg + 4, sec);
    put32(msg + 8, nsec);
    uint8_t* f = msg + h.bytes;
    put32(f + 0, __float_as_uint(0.0f));                             // angle_min
    put32(f + 4, __float_as_uint((float)(2.0 * 3.14159265358979323846)));  // angle_max
    put32(f + 8, __float_as_uint(a.angle_increment[i]));
    put32(f + 12, __float_as_uint(__double2float_rn(d / denom)));    // time_increment
    put32(f + 16, __float_as_uint(__double2float_rn(d)));            // scan_time
    put32(f + 20, __float_as_uint(0.15f));                           // range_min
    put32(f + 24, __float_as_uint(h.range_max));
    put32(f + 28, n);
    put32(msg + P + 4 * (size_t)n, n);  // intensities count
  }
}

__global__ void __launch_bounds__(CT) laserscan_msgs_kernel(MsgWriteArgs a) {
  const uint32_t i = a.slot0 + blockIdx.y;
  const uint32_t size = a.sizes[i];
  if (size == 0) return;
  const uint32_t n = a.counts[i];
  const StreamMsgHeader& h = a.hdr[i / a.max_scans];
  const uint32_t P = h.bytes + 32;  // the 7 floats and the ranges count follow the header
  uint8_t* msg = a.out + (a.offsets[i] - a.out_base);
  if (blockIdx.x == 0) put_laserscan_fixed<CT>(a, i, n, h, P, msg);
  uint32_t* r_out = reinterpret_cast<uint32_t*>(msg + P);
  uint32_t* i_out = r_out + n + 1;
  const uint32_t* r_in = reinterpret_cast<const uint32_t*>(a.ranges + (size_t)i * a.stride);
  const uint32_t* i_in = reinterpret_cast<const uint32_t*>(a.intensities + (size_t)i * a.stride);
  for (uint32_t j = blockIdx.x * CT + threadIdx.x; j < n; j += gridDim.x * CT) {
    r_out[j] = __ldg(r_in + j);
    i_out[j] = __ldg(i_in + j);
  }
}

__global__ void __launch_bounds__(CT) pointcloud2_msgs_kernel(MsgWriteArgs a, CloudTail t) {
  const uint32_t i = a.slot0 + blockIdx.y;
  const uint32_t size = a.sizes[i];
  if (size == 0) return;
  const uint32_t n = a.counts[i];
  const StreamMsgHeader& h = a.hdr[i / a.max_scans];
  const uint32_t P = h.bytes + t.bytes;  // ends with the data length
  uint8_t* msg = a.out + (a.offsets[i] - a.out_base);
  if (blockIdx.x == 0) {
    put_header<CT>(msg, h);
    for (uint32_t w = threadIdx.x; w < t.bytes / 4; w += CT) {
      const uint32_t v = w == t.at_width ? n : (w == t.at_row_step || w == t.at_data) ? 16u * n : t.w[w];
      put32(msg + h.bytes + 4 * w, v);
    }
    if (threadIdx.x == 0) {
      uint32_t sec, nsec;
      msg_stamp(a.begin_us ? a.begin_us[i] : 0ull, a.clock_offset_ns, &sec, &nsec);
      put32(msg + 4, sec);
      put32(msg + 8, nsec);
      msg[P + 16 * (size_t)n] = 1;  // is_dense: the cloud path drops unmeasured points
    }
  }
  const uint4* d_in = reinterpret_cast<const uint4*>(a.xyzi + (size_t)i * a.stride * 4);
  if ((P & 15u) == 0) {  // the message starts 16-aligned: the data is 16-aligned iff P is
    uint4* d_out = reinterpret_cast<uint4*>(msg + P);
    for (uint32_t j = blockIdx.x * CT + threadIdx.x; j < n; j += gridDim.x * CT) d_out[j] = __ldg(d_in + j);
  } else {
    uint32_t* o = reinterpret_cast<uint32_t*>(msg + P);
    const uint32_t* in = reinterpret_cast<const uint32_t*>(d_in);
    for (uint32_t j = blockIdx.x * CT + threadIdx.x; j < 4 * n; j += gridDim.x * CT) o[j] = __ldg(in + j);
  }
}

// ---- messages written by a push --------------------------------------------------------------------------------
// One CTA over the chunk's slots in tiles of MT, as msg_table_kernel, the carry passing from tile to tile and, through
// *a.carry, from chunk to chunk: the chunks of a push run one after the other (one stream, or the host push's lanes
// ordered by an event), so each reads the end the one before it wrote.
// K = kLaserScan: a published slot's bound, its message at the view's node count rounded up to 16, places it before
// the scan kernels run (place[i]); the end of the bounds is the total.
// K = kPointCloud2: a published slot's exact size at its cloud's point count, once the cloud kernels have run, rounded
// up to 16 for the offsets (msg_table_kernel's packing); sizes[i] is the size when the message fits capacity, else 0,
// and the total is the end of the last message, carried in carry[1].
template <MsgKind K>
__global__ void __launch_bounds__(MT) push_msg_dir_kernel(PushMsgDirArgs a) {
  constexpr bool kCloud = K == MsgKind::kPointCloud2;
  __shared__ unsigned long long s_warp[MT / 32];
  __shared__ unsigned long long s_first, s_fit_end, s_last_end;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    s_first = a.first ? 0ull : *a.carry;
    s_fit_end = s_first;
    if constexpr (kCloud) s_last_end = a.first ? 0ull : a.carry[1];
  }
  __syncthreads();
  const unsigned long long first = s_first, rel = a.rebase ? first : 0ull;
  unsigned long long carry = first;
  for (uint32_t t0 = 0; t0 < a.n_slots; t0 += MT) {
    const uint32_t i = t0 + tid;
    uint32_t bound = 0, hb = 0;  // PointCloud2: the exact size
    if (i < a.n_slots) {
      const uint32_t s = i / a.max_scans, k = i - s * a.max_scans;
      hb = a.hdr[s].bytes;
      const bool off = kCloud && a.clouds && a.clouds[s].route == kCloudOff;  // a stream without a cloud
      if (k < min(a.scans_per_stream[s], a.max_scans) && !off) {
        if constexpr (kCloud) bound = msg_bytes(K, hb, a.counts[i]);
        else bound = (msg_bytes(K, hb, a.views[i].y) + 15u) & ~15u;
      }
    }
    const unsigned long long v = kCloud ? (bound + 15u) & ~15u : bound;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= (uint32_t)o) inc += u;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long base = 0, tile = 0;
    for (uint32_t w = 0; w < MT / 32; ++w) {
      const unsigned long long x = s_warp[w];
      if (w < warp) base += x;
      tile += x;
    }
    const unsigned long long off = carry + base + inc - v;
    if (i < a.n_slots) {
      const bool fits = bound != 0 && off + bound <= a.capacity;
      a.offsets[i] = off;
      if constexpr (kCloud) {
        a.sizes[i] = fits ? bound : 0u;
        if (bound) atomicMax(&s_last_end, off + bound);
      } else {
        a.place[i] = fits ? off - rel + hb + 32u : kOutSkip;
      }
      if (fits) atomicMax(&s_fit_end, off + bound);
    }
    carry += tile;
    __syncthreads();  // s_warp is rewritten by the next tile
  }
  if (tid == 0) {
    *a.carry = carry;
    const unsigned long long end = kCloud ? s_last_end : carry;
    if constexpr (kCloud) a.carry[1] = end;
    if (a.extent) {
      a.extent[0] = first;
      a.extent[1] = s_fit_end;
      a.extent[2] = end;
    }
    if (a.total) *a.total = end;
  }
}

// one CTA of 32 threads per slot: the arrays are the scan kernels'
__global__ void __launch_bounds__(32) laserscan_placed_kernel(MsgWriteArgs a, const unsigned long long* place,
                                                              uint32_t* sizes) {
  const uint32_t i = blockIdx.x;
  const unsigned long long pl = place[i];
  const uint32_t n = (pl & kOutSkip) ? 0u : a.counts[i];
  const StreamMsgHeader& h = a.hdr[i / a.max_scans];
  if (threadIdx.x == 0) sizes[i] = n ? msg_bytes(MsgKind::kLaserScan, h.bytes, n) : 0u;
  if (n == 0) return;
  const uint32_t P = h.bytes + 32;
  put_laserscan_fixed<32>(a, i, n, h, P, a.out + (pl - P));
}

}  // namespace

cudaError_t launch_push_msg_dir(const PushMsgDirArgs& a, MsgKind kind, cudaStream_t stream) {
  if (kind == MsgKind::kLaserScan)
    push_msg_dir_kernel<MsgKind::kLaserScan><<<1, MT, 0, stream>>>(a);
  else
    push_msg_dir_kernel<MsgKind::kPointCloud2><<<1, MT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_laserscan_placed(const MsgWriteArgs& a, const unsigned long long* place, uint32_t* sizes,
                                    cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  laserscan_placed_kernel<<<a.n, 32, 0, stream>>>(a, place, sizes);
  return cudaGetLastError();
}

cudaError_t launch_msg_table(const MsgTableArgs& a, cudaStream_t stream) {
  if (a.n_slots == 0) return cudaSuccess;
  msg_table_kernel<<<1, MT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_laserscan_msgs(const MsgWriteArgs& a, uint32_t max_beams, cudaStream_t stream) {
  const uint32_t bx = std::max(1u, std::min((max_beams + CT * 4 - 1) / (CT * 4), 32u));
  for (uint32_t k = 0; k < a.n; k += 65535) {
    MsgWriteArgs b = a;
    b.slot0 = a.slot0 + k;
    laserscan_msgs_kernel<<<dim3(bx, std::min(65535u, a.n - k)), CT, 0, stream>>>(b);
  }
  return cudaGetLastError();
}

cudaError_t launch_pointcloud2_msgs(const MsgWriteArgs& a, const CloudTail& t, uint32_t max_points,
                                    cudaStream_t stream) {
  const uint32_t bx = std::max(1u, std::min((max_points + CT * 4 - 1) / (CT * 4), 32u));
  for (uint32_t k = 0; k < a.n; k += 65535) {
    MsgWriteArgs b = a;
    b.slot0 = a.slot0 + k;
    pointcloud2_msgs_kernel<<<dim3(bx, std::min(65535u, a.n - k)), CT, 0, stream>>>(b, t);
  }
  return cudaGetLastError();
}

cudaError_t launch_laserscan_cdr(const LaserScanCdrArgs& a, const CdrTemplate& t, cudaStream_t stream) {
  if (a.n_scans == 0) return cudaSuccess;
  const uint32_t bx = std::max(1u, std::min((a.stride + CT * 4 - 1) / (CT * 4), 32u));
  for (uint32_t s0 = 0; s0 < a.n_scans; s0 += 65535) {
    LaserScanCdrArgs b = a;
    b.meta += s0;
    b.ranges += (size_t)s0 * a.stride;
    b.intensities += (size_t)s0 * a.stride;
    b.beam_counts += s0;
    if (b.angle_increment) b.angle_increment += s0;
    b.cdr_out += (size_t)s0 * a.cdr_stride;
    if (b.cdr_sizes) b.cdr_sizes += s0;
    laserscan_cdr_kernel<<<dim3(bx, std::min(65535u, a.n_scans - s0)), CT, 0, stream>>>(b, t);
  }
  return cudaGetLastError();
}

cudaError_t launch_pointcloud2_cdr(const PointCloudCdrArgs& a, const CdrTemplate& t, cudaStream_t stream) {
  if (a.n_clouds == 0) return cudaSuccess;
  const uint32_t bx = std::max(1u, std::min((a.stride + CT * 4 - 1) / (CT * 4), 32u));
  for (uint32_t s0 = 0; s0 < a.n_clouds; s0 += 65535) {
    PointCloudCdrArgs b = a;
    b.stamps += 2 * (size_t)s0;
    b.xyzi += (size_t)s0 * a.stride * 4;
    b.point_counts += s0;
    b.cdr_out += (size_t)s0 * a.cdr_stride;
    if (b.cdr_sizes) b.cdr_sizes += s0;
    pointcloud2_cdr_kernel<<<dim3(bx, std::min(65535u, a.n_clouds - s0)), CT, 0, stream>>>(b, t);
  }
  return cudaGetLastError();
}

}  // namespace rpl
