// session_nodes.cu -- the grabbed-node buffers of a stream session's last push (rpl_*_stream_nodes[_dev]): what
// RealLidarDriver::grab_scan_data returns for each scan the push published (reference lidar_driver_wrapper.cpp:307-342),
// packed one behind the other.  A buffer's size is its view's count, known before any scan kernel runs: the directory
// kernel here computes every buffer's position first, the scan kernels then write each ascended revolution straight
// to its position (ScanBatchArgs::out_first), and the gather kernel copies the revolutions that are not ascended.
#include <algorithm>

#include "rpl_device.cuh"
#include "scan_args.h"
#include "session_nodes_args.h"

namespace rpl {
namespace {

constexpr int DT = 1024;  // the directory: one CTA
constexpr int GT = 256;   // the gather: one CTA per slot at a time

// The slots in tiles of DT: the exclusive scan of the counts rounded up to even, the carry passing from tile to tile,
// and the end of the last buffer; then, knowing whether the buffers fit, every slot's count, place and status.
__global__ void __launch_bounds__(DT) node_directory_kernel(NodeDirArgs a) {
  __shared__ unsigned long long s_warp[DT / 32];
  __shared__ unsigned long long s_end;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_end = 0;
  unsigned long long carry = 0;
  for (uint32_t t0 = 0; t0 < a.n_slots; t0 += DT) {
    const uint32_t i = t0 + tid;
    const uint32_t n = i < a.n_slots ? a.views[i].y : 0u;
    const unsigned long long v = (n + 1u) & ~1u;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= (uint32_t)o) inc += u;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long base = 0, tile = 0;
    for (uint32_t w = 0; w < DT / 32; ++w) {
      const unsigned long long x = s_warp[w];
      if (w < warp) base += x;
      tile += x;
    }
    const unsigned long long off = carry + base + inc - v;
    if (i < a.n_slots) {
      a.offsets[i] = off;
      if (n) atomicMax(&s_end, off + n);
    }
    carry += tile;
    __syncthreads();  // s_warp is rewritten by the next tile; the offsets are visible to the whole CTA
  }
  const unsigned long long total = s_end;
  const bool fits = total <= a.capacity;
  for (uint32_t i = tid; i < a.n_slots; i += DT) {
    const uint32_t n = fits ? a.views[i].y : 0u;
    a.counts[i] = n;
    unsigned long long place = ~0ull;
    if (n) {
      const bool ascended = a.ascend ? a.ascend[i / a.max_scans] != 0 : a.ascend_all != 0;
      const unsigned long long first = a.rebase ? a.offsets[i - i % a.chunk_slots] : 0ull;
      place = (a.offsets[i] - first) | (ascended ? 0ull : kOutSkip);
    }
    a.place[i] = place;
    if (place & kOutSkip) a.status[i] = kResultOk;
  }
  if (tid == 0) *a.total = total;
}

// A view may start on an odd node of the arena; its buffer never does.  Two nodes per thread where both sides are
// 16-byte aligned, one otherwise.
__global__ void __launch_bounds__(GT) node_gather_kernel(NodeGatherArgs a) {
  for (uint32_t s = blockIdx.x; s < a.n_slots; s += gridDim.x) {
    const unsigned long long place = a.place[s];
    if (!(place & kOutSkip) || place == ~0ull) continue;
    const uint2 view = a.views[s];
    const uint2* src = a.nodes + view.x;
    uint2* dst = a.out + (place & ~kOutSkip);
    const uint32_t n = view.y;
    if ((view.x & 1u) == 0) {
      const uint4* s4 = reinterpret_cast<const uint4*>(src);
      uint4* d4 = reinterpret_cast<uint4*>(dst);
      for (uint32_t w = threadIdx.x; w < n / 2; w += GT) d4[w] = __ldg(s4 + w);
      if ((n & 1u) && threadIdx.x == 0) dst[n - 1] = __ldg(src + n - 1);
    } else {
      for (uint32_t i = threadIdx.x; i < n; i += GT) dst[i] = __ldg(src + i);
    }
  }
}

}  // namespace

cudaError_t launch_node_directory(const NodeDirArgs& a, cudaStream_t stream) {
  node_directory_kernel<<<1, DT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_node_gather(const NodeGatherArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n_slots == 0) return cudaSuccess;
  const int grid = (int)std::min<uint32_t>(a.n_slots, (uint32_t)num_sms * 8u);
  node_gather_kernel<<<grid, GT, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rpl
