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
//
// rescan_window_kernel (DESIGN.md 5.7.1 "Windows over the re-gridded scans"), the push form's streams with a window:
// laser_filters' LaserArrayFilter over the same grids, a per-bin median or mean of each stream's last revolutions, whose
// definition and CPU restatement is oracle/rescan_window_oracle.py.  It runs behind rescan_kernel, reads each grid from
// the message rescan_kernel wrote (or builds it with the same loop, rescan_slot_grid, when the message did not fit),
// writes W over it, and keeps the last observations - 1 grids of the stream in a ring in device memory.
//
// The merged scans (DESIGN.md 5.7.1 "Merged scans from the push"), a scan merger over the same grids, whose definition
// and CPU restatement is oracle/rescan_merge_oracle.py: rescan_hold_kernel keeps each grouped stream's newest written
// re-grid message's ranges and stamp in its held row, per chunk behind the window kernel; at the end of the push
// rescan_merge_dir_kernel places one message per group that has news and rescan_merge_kernel writes it, the per-bin
// minimum of the contributors' held rows (merge_bins, shared with the stateless rescan_merge_batch_kernel).
#include <algorithm>

#include "beam_point.cuh"
#include "msg_fixed.cuh"
#include "rescan_args.h"
#include "scan_cloud_point.cuh"

namespace rpl {
namespace {

constexpr int RT = 256;

// Slot i's grid in s_bins, by the RT threads of the CTA: every bin seeded, then the least range of the points that land
// in it; s_bins is complete when this returns
__device__ __forceinline__ void rescan_slot_grid(const ScanCloudArgs& c, uint32_t i, const RescanGrid& g,
                                                 uint32_t* s_bins) {
  const uint32_t tid = threadIdx.x;
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
}

// The re-grid message's members behind its header, by threads 0 .. 7: angle_min, angle_max, angle_increment,
// time_increment 0, scan_time, range_min, range_max, the ranges' count
__device__ __forceinline__ void put_rescan_fields(uint8_t* body, const RescanGrid& g) {
  const uint32_t tid = threadIdx.x;
  if (tid < 8) {
    const float f = tid == 0 ? g.angle_min : tid == 1 ? g.angle_max : tid == 2 ? g.angle_increment
                    : tid == 4 ? g.scan_time : tid == 5 ? g.range_min : tid == 6 ? g.range_max : 0.0f;
    put32(body + 4 * tid, tid == 7 ? g.bins : __float_as_uint(f));
  }
}

__global__ void __launch_bounds__(RT) rescan_kernel(const __grid_constant__ RescanArgs a) {
  __shared__ uint32_t s_bins[kRescanMaxBins];
  const ScanCloudArgs& c = a.c;
  const uint32_t tid = threadIdx.x;
  for (uint32_t s = blockIdx.x; s < c.m.n; s += gridDim.x) {
    const uint32_t i = c.m.slot0 + s;
    if (c.m.out && c.m.sizes[i] == 0) continue;  // no message, or the messages do not fit
    const RescanGrid& g = a.grid ? a.grid[i / c.m.max_scans] : a.grid_one;
    rescan_slot_grid(c, i, g, s_bins);
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
      put_rescan_fields(body, g);
      for (uint32_t b = tid; b < g.bins; b += RT) put32(body + 32 + 4 * b, s_bins[b]);
    } else {
      uint32_t* row = reinterpret_cast<uint32_t*>(a.out) + (size_t)i * g.bins;
      for (uint32_t b = tid; b < g.bins; b += RT) row[b] = s_bins[b];
    }
    __syncthreads();  // s_bins is seeded again for the next slot
  }
}

// W (oracle/rescan_window_oracle.py) of the n values v[0 .. n) of one bin, oldest first, 1 <= n <= kRescanWindowMax;
// v[j] for j >= n is not read.  Median: the value v[j] with at most k = (n - 1) / 2 values below it and more than k at
// or below it -- a value itself, whatever the ties -- in n * n comparisons.  Mean: the float sum from +0 oldest first,
// over n.  The loops are unrolled and leave at n (the same for every thread of the CTA), so every index is a constant
// and v stays in registers.
__device__ __forceinline__ float window_stat(const float (&v)[kRescanWindowMax], uint32_t n, uint32_t statistic) {
  if (statistic == kRescanWindowMean) {
    float sum = 0.0f;
#pragma unroll
    for (uint32_t j = 0; j < kRescanWindowMax; ++j) {
      if (j >= n) break;
      sum = __fadd_rn(sum, v[j]);
    }
    return __fdiv_rn(sum, (float)n);
  }
  const uint32_t k = (n - 1) / 2;
  float m = v[0];
#pragma unroll
  for (uint32_t j = 0; j < kRescanWindowMax; ++j) {
    if (j >= n) break;
    uint32_t lt = 0, le = 0;
#pragma unroll
    for (uint32_t q = 0; q < kRescanWindowMax; ++q) {
      if (q >= n) break;
      lt += v[q] < v[j] ? 1u : 0u;
      le += v[q] <= v[j] ? 1u : 0u;
    }
    if (lt <= k && k < le) m = v[j];
  }
  return m;
}

// One CTA per stream with a window (RescanWindowArgs), its slots in revolution order; each thread keeps the same bins
// from the grid through the ring to the message, so the ring needs no barrier of its own
__global__ void __launch_bounds__(RT) rescan_window_kernel(const __grid_constant__ RescanWindowArgs a) {
  __shared__ uint32_t s_bins[kRescanMaxBins];
  const ScanCloudArgs& c = a.r.c;
  const uint32_t tid = threadIdx.x;
  for (uint32_t q = blockIdx.x; q < a.n; q += gridDim.x) {
    const uint32_t s = a.streams[q] - a.stream0;
    const RescanGrid& g = a.r.grid[s];
    const RescanWindow w = a.win[s];
    const uint32_t R = w.observations - 1, bins = g.bins;
    float* ring = a.ring + w.ring;
    uint2 st = a.state[s];  // {held, next row}
    for (uint32_t k = 0; k < c.m.max_scans; ++k) {
      const uint32_t i = s * c.m.max_scans + k;
      if (c.scan_sizes[i] == 0) continue;  // no LaserScan message: not a revolution of the window
      // the message rescan_kernel has just written holds the grid; one that did not fit is built here
      uint8_t* ranges = nullptr;
      if (c.m.sizes[i]) {
        const StreamMsgHeader& h = c.transform ? c.cloud_hdr[i / c.m.max_scans] : c.m.hdr[i / c.m.max_scans];
        ranges = c.m.out + (c.m.offsets[i] - c.m.out_base) + h.bytes + 32;
      } else {
        rescan_slot_grid(c, i, g, s_bins);
      }
      const uint32_t n = st.x + 1;
      uint32_t row[kRescanWindowMax - 1];  // the held values' rows, oldest first
#pragma unroll
      for (uint32_t j = 0; j + 1 < kRescanWindowMax; ++j) row[j] = (st.y + R - st.x + j) % R;
      for (uint32_t b = tid; b < bins; b += RT) {
        const float x = __uint_as_float(ranges ? *reinterpret_cast<const uint32_t*>(ranges + 4 * b) : s_bins[b]);
        float v[kRescanWindowMax];
#pragma unroll
        for (uint32_t j = 0; j < kRescanWindowMax; ++j)
          v[j] = j < st.x ? ring[(size_t)row[j < kRescanWindowMax - 1 ? j : 0] * bins + b]
                 : x;  // v[st.x], the newest; entries past it are not read
        if (ranges) put32(ranges + 4 * b, __float_as_uint(window_stat(v, n, w.statistic)));
        ring[(size_t)st.y * bins + b] = x;
      }
      st.x = min(st.x + 1, R);
      st.y = st.y + 1 == R ? 0u : st.y + 1;
      __syncthreads();  // s_bins is seeded again for the next slot
    }
    if (tid == 0) a.state[s] = st;
  }
}

// one thread per (row, bin) of the stateless form
__global__ void __launch_bounds__(RT) rescan_window_batch_kernel(const float* __restrict__ in, uint32_t n_scans,
                                                                 uint32_t bins, uint32_t observations,
                                                                 uint32_t statistic, float* __restrict__ out) {
  const unsigned long long total = (unsigned long long)n_scans * bins;
  for (unsigned long long e = blockIdx.x * (unsigned long long)RT + threadIdx.x; e < total;
       e += (unsigned long long)gridDim.x * RT) {
    const uint32_t t = (uint32_t)(e / bins), b = (uint32_t)(e - (unsigned long long)t * bins);
    const uint32_t n = min(observations, t + 1), first = t + 1 - n;
    float v[kRescanWindowMax];
#pragma unroll
    for (uint32_t j = 0; j < kRescanWindowMax; ++j)
      v[j] = j < n ? __ldg(in + (size_t)(first + j) * bins + b) : 0.0f;  // past n: not read
    out[e] = window_stat(v, n, statistic);
  }
}

// M (oracle/rescan_merge_oracle.py) at bin b: the least of the bits m and bin b of every row row(j), j < n, that is not
// null.  Re-grid values are >= +0 and never NaN, so the unsigned min of the bits is the float min, in any order.
template <class Row>
__device__ __forceinline__ uint32_t merge_bins(uint32_t m, uint32_t n, uint32_t b, Row row) {
  for (uint32_t j = 0; j < n; ++j)
    if (const float* r = row(j)) m = min(m, __float_as_uint(r[b]));
  return m;
}

// One CTA per grouped stream of the chunk (RescanHoldArgs)
__global__ void __launch_bounds__(RT) rescan_hold_kernel(const __grid_constant__ RescanHoldArgs a) {
  const ScanCloudArgs& c = a.r.c;
  const uint32_t tid = threadIdx.x;
  for (uint32_t q = blockIdx.x; q < a.n; q += gridDim.x) {
    const uint32_t s = a.streams[q] - a.stream0;
    uint32_t i = kRescanMergeNone;  // the newest slot whose re-grid message was written
    for (uint32_t k = c.m.max_scans; k-- > 0;)
      if (c.m.sizes[s * c.m.max_scans + k]) {
        i = s * c.m.max_scans + k;
        break;
      }
    if (i == kRescanMergeNone) continue;  // the held grid stays as it was
    const StreamMsgHeader& h = c.transform ? c.cloud_hdr[s] : c.m.hdr[s];
    const uint8_t* msg = c.m.out + (c.m.offsets[i] - c.m.out_base);
    const uint32_t* ranges = reinterpret_cast<const uint32_t*>(msg + h.bytes + 32);
    float* row = a.rows + (size_t)a.row[s] * kRescanMaxBins;
    for (uint32_t b = tid; b < a.r.grid[s].bins; b += RT) row[b] = __uint_as_float(ranges[b]);
    if (tid == 0)
      a.held[s] = RescanHeld{*reinterpret_cast<const uint32_t*>(msg + 4), *reinterpret_cast<const uint32_t*>(msg + 8),
                             a.seq, c.transform ? kHeldTargetHdr : kHeldScanHdr};
  }
}

__device__ __forceinline__ bool contributes(const RescanMergeArgs& a, const RescanHeld& h, uint32_t g) {
  return h.hdr && a.seq - h.seq <= a.max_age[g];
}

// the header stream s's held grid's message took
__device__ __forceinline__ const StreamMsgHeader& held_header(const RescanMergeArgs& a, uint32_t s) {
  return (a.held[s].hdr == kHeldTargetHdr ? a.hdr_target : a.hdr_scan)[s];
}

// One CTA over the groups in tiles of RT, as push_msg_dir_kernel over slots
__global__ void __launch_bounds__(RT) rescan_merge_dir_kernel(const __grid_constant__ RescanMergeArgs a) {
  __shared__ unsigned long long s_warp[RT / 32];
  __shared__ unsigned long long s_fit_end, s_last_end;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_fit_end = s_last_end = 0;
  __syncthreads();
  unsigned long long carry = 0;
  for (uint32_t g0 = 0; g0 < a.n_groups; g0 += RT) {
    const uint32_t g = g0 + tid;
    uint32_t size = 0;
    if (g < a.n_groups) {
      bool publish = false;
      uint32_t pick = kRescanMergeNone, sec = 0, nsec = 0;
      for (uint32_t j = a.begin[g]; j < a.begin[g + 1]; ++j) {  // ascending: a tie keeps the lowest index
        const uint32_t s = a.members[j];
        const RescanHeld h = a.held[s];
        if (!contributes(a, h, g)) continue;
        publish |= h.seq == a.seq;
        if (pick == kRescanMergeNone || h.sec > sec || (h.sec == sec && h.nanosec > nsec)) {
          pick = s;
          sec = h.sec;
          nsec = h.nanosec;
        }
      }
      if (!publish) pick = kRescanMergeNone;
      else size = held_header(a, pick).bytes + 36u + 4u * a.grid[pick].bins;
      a.pick[g] = pick;
    }
    const unsigned long long v = (size + 15u) & ~15u;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= (uint32_t)o) inc += u;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long base = 0, tile = 0;
    for (uint32_t w = 0; w < RT / 32; ++w) {
      const unsigned long long x = s_warp[w];
      if (w < warp) base += x;
      tile += x;
    }
    const unsigned long long off = carry + base + inc - v;
    if (g < a.n_groups) {
      const bool fits = size != 0 && off + size <= a.capacity;
      a.offsets[g] = off;
      a.sizes[g] = fits ? size : 0u;
      if (size) atomicMax(&s_last_end, off + size);
      if (fits) atomicMax(&s_fit_end, off + size);
    }
    carry += tile;
    __syncthreads();  // s_warp is rewritten by the next tile
  }
  if (tid == 0) {
    *a.total = s_last_end;
    if (a.fit_end) *a.fit_end = s_fit_end;
  }
}

// One CTA per group whose message the directory placed and that fits
__global__ void __launch_bounds__(RT) rescan_merge_kernel(const __grid_constant__ RescanMergeArgs a) {
  const uint32_t tid = threadIdx.x;
  for (uint32_t g = blockIdx.x; g < a.n_groups; g += gridDim.x) {
    if (a.sizes[g] == 0) continue;
    const uint32_t p = a.pick[g];
    const StreamMsgHeader& h = held_header(a, p);
    const RescanGrid& gr = a.grid[p];
    uint8_t* msg = a.out + a.offsets[g];
    put_header<RT>(msg, h);
    uint8_t* body = msg + h.bytes;
    if (tid == 0) {
      const RescanHeld x = a.held[p];
      put32(msg + 4, x.sec);
      put32(msg + 8, x.nanosec);
      put32(body + 32 + 4 * gr.bins, 0u);  // intensities: none
    }
    put_rescan_fields(body, gr);
    const uint32_t j0 = a.begin[g], n = a.begin[g + 1] - j0;
    for (uint32_t b = tid; b < gr.bins; b += RT)
      put32(body + 32 + 4 * b, merge_bins(gr.seed, n, b, [&](uint32_t j) -> const float* {
              const uint32_t s = a.members[j0 + j];
              return contributes(a, a.held[s], g) ? a.rows + (size_t)a.row[s] * kRescanMaxBins : nullptr;
            }));
  }
}

// one thread per (group, bin) of the stateless form
__global__ void __launch_bounds__(RT) rescan_merge_batch_kernel(const float* __restrict__ in,
                                                                const uint32_t* __restrict__ row_group, uint32_t n_rows,
                                                                uint32_t n_groups, uint32_t bins, uint32_t seed,
                                                                float* __restrict__ out) {
  const unsigned long long total = (unsigned long long)n_groups * bins;
  for (unsigned long long e = blockIdx.x * (unsigned long long)RT + threadIdx.x; e < total;
       e += (unsigned long long)gridDim.x * RT) {
    const uint32_t g = (uint32_t)(e / bins), b = (uint32_t)(e - (unsigned long long)g * bins);
    out[e] = __uint_as_float(merge_bins(seed, n_rows, b, [&](uint32_t r) -> const float* {
      return __ldg(row_group + r) == g ? in + (size_t)r * bins : nullptr;
    }));
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

cudaError_t launch_rescan_window(const RescanWindowArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  static const int k = [] {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, rescan_window_kernel, RT, 0);
    return std::max(n, 1);
  }();
  rescan_window_kernel<<<(int)std::min<uint32_t>(a.n, (uint32_t)(num_sms * k)), RT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_rescan_window_batch(const float* in, uint32_t n_scans, uint32_t bins, uint32_t observations,
                                       uint32_t statistic, float* out, int num_sms, cudaStream_t stream) {
  const unsigned long long total = (unsigned long long)n_scans * bins;
  if (total == 0) return cudaSuccess;
  const unsigned long long blocks = std::min<unsigned long long>((total + RT - 1) / RT, (unsigned long long)num_sms * 8);
  rescan_window_batch_kernel<<<(unsigned)blocks, RT, 0, stream>>>(in, n_scans, bins, observations, statistic, out);
  return cudaGetLastError();
}

cudaError_t launch_rescan_hold(const RescanHoldArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  rescan_hold_kernel<<<(int)std::min<uint32_t>(a.n, (uint32_t)num_sms * 8u), RT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_rescan_merge(const RescanMergeArgs& a, int num_sms, cudaStream_t stream) {
  rescan_merge_dir_kernel<<<1, RT, 0, stream>>>(a);
  if (a.n_groups) rescan_merge_kernel<<<(int)std::min<uint32_t>(a.n_groups, (uint32_t)num_sms * 8u), RT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_rescan_merge_batch(const float* in, const uint32_t* row_group, uint32_t n_rows, uint32_t n_groups,
                                      uint32_t bins, uint32_t seed, float* out, int num_sms, cudaStream_t stream) {
  const unsigned long long total = (unsigned long long)n_groups * bins;
  if (total == 0) return cudaSuccess;
  const unsigned long long blocks = std::min<unsigned long long>((total + RT - 1) / RT, (unsigned long long)num_sms * 8);
  rescan_merge_batch_kernel<<<(unsigned)blocks, RT, 0, stream>>>(in, row_group, n_rows, n_groups, bins, seed, out);
  return cudaGetLastError();
}

}  // namespace rpl
