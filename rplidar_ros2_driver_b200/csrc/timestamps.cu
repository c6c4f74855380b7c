// timestamps.cu -- per-sample timestamps (SURVEY.md 8(f) rank 4).
//
// The SDK stamps every decoded node with "receive time of a capsule minus a delay model" (delay_model.cuh); the node
// then throws all but the scan-begin stamp away (src/rplidar_node.cpp:417,442).  Here the stamps are a function of the
// decoder's per-capsule report: one thread per node slot, 8 bytes written per node, nothing read but the capsule's
// status/offset/rx words (shared by the 32..96 threads of a capsule).
#include "decode_args.h"
#include "delay_model.cuh"
#include "rpl_device.cuh"

namespace rpl {

namespace {

__global__ void node_timestamps_kernel(TimestampArgs a, DelayModel m) {
  const uint32_t s = blockIdx.y;
  const uint32_t n_caps = a.capsule_counts[s];
  const size_t cbase = (size_t)s * a.stride_capsules;
  unsigned long long* out = a.node_ts_us + cbase * m.per;
  const uint32_t slots = n_caps * m.per;
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += gridDim.x * blockDim.x) {
    const uint32_t j = q / m.per, pos = q - j * m.per;
    if (!(a.capsule_status[cbase + j] & 4u)) continue;  // RPL_CAPSULE_EMIT
    const unsigned long long rx = a.capsule_rx_us[cbase + j - (m.prev_base ? 1u : 0u)];
    unsigned long long d = m.base;
    if (m.group >= 0) d += (unsigned long long)(m.group - (int)pos) * m.sd;
    out[a.capsule_node_offset[cbase + j] + pos] = rx - d;
  }
}

__global__ void normal_timestamps_kernel(NormalTimestampArgs a, unsigned long long delay) {
  const uint32_t s = blockIdx.y;
  const uint32_t n = a.node_counts[s];
  const uint32_t* ends = a.node_end + (size_t)s * a.stride_nodes;
  const unsigned long long* rx = a.chunk_rx_us + (size_t)s * a.stride_chunks;
  unsigned long long* out = a.node_ts_us + (size_t)s * a.stride_nodes;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = rx[ends[i] / a.chunk_bytes] - delay;
}

}  // namespace

cudaError_t launch_node_timestamps(uint32_t ans_type, const TimingDesc& t, const TimestampArgs& a,
                                   cudaStream_t stream) {
  if (a.n_streams == 0 || a.stride_capsules == 0) return cudaSuccess;
  const DelayModel m = delay_model(ans_type, t);
  const uint32_t slots = a.stride_capsules * m.per;
  const uint32_t bx = std::min<uint32_t>((slots + 1023) / 1024, 64u);
  for (uint32_t s0 = 0; s0 < a.n_streams; s0 += 65535) {
    TimestampArgs b = a;
    const size_t cb = (size_t)s0 * a.stride_capsules;
    b.capsule_rx_us += cb;
    b.capsule_status += cb;
    b.capsule_node_offset += cb;
    b.capsule_counts += s0;
    b.node_ts_us += cb * m.per;
    node_timestamps_kernel<<<dim3(bx, std::min<uint32_t>(65535u, a.n_streams - s0)), 256, 0, stream>>>(b, m);
  }
  return cudaGetLastError();
}

cudaError_t launch_normal_timestamps(const TimingDesc& t, const NormalTimestampArgs& a, cudaStream_t stream) {
  if (a.n_streams == 0 || a.stride_nodes == 0) return cudaSuccess;
  const DelayModel m = delay_model(0x81, t);
  const uint32_t bx = std::min<uint32_t>((a.stride_nodes + 1023) / 1024, 64u);
  for (uint32_t s0 = 0; s0 < a.n_streams; s0 += 65535) {
    NormalTimestampArgs b = a;
    b.node_end += (size_t)s0 * a.stride_nodes;
    b.node_counts += s0;
    b.chunk_rx_us += (size_t)s0 * a.stride_chunks;
    b.node_ts_us += (size_t)s0 * a.stride_nodes;
    normal_timestamps_kernel<<<dim3(bx, std::min<uint32_t>(65535u, a.n_streams - s0)), 256, 0, stream>>>(b, m.base);
  }
  return cudaGetLastError();
}

}  // namespace rpl
