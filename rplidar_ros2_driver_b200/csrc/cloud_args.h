// cloud_args.h -- workspace and launchers of the PointCloud2 post-processing (see cloud.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lidar_args.h"

namespace rpl {

struct CloudWorkspace {
  float2* trig = nullptr;        // [65536] (cos, sin) of angle_rad(key), rounded from double
  float2* angle = nullptr;       // [65536] (angle_rad, inverted angle) exactly as publish_scan forms them
  void* scratch = nullptr;       // per-CTA staging, see cloud.cu
  size_t scratch_per_cta = 0;
  uint32_t max_nodes = 0;
  int ctas = 0;
};

cudaError_t cloud_configure();
cudaError_t cloud_workspace_alloc(CloudWorkspace& ws, int num_sms, uint32_t max_nodes);
void cloud_workspace_free(CloudWorkspace& ws);
// Per-stream clouds (ScanBatchArgs::clouds) in a post pass: scan s is served iff cloud_route(at[s / per], launches)
// == route and its entry has the step, which then takes its sor_k / sor_alpha / voxel from there.  at == nullptr:
// every scan, with the pass's own parameters.
struct CloudTable {
  const CloudSettings* at;
  uint32_t per, launches, route;
};
// steps 4-5 (SOR, voxel grid) over per-scan clouds already in angle order, in place.  list / list_count
// (device, nullable): restrict the pass to these scans (what the shared-memory kernel of scan_small.cu
// handed to the general kernel); the general path for revolutions above 4096 nodes.  With tab.at: sor_k > 0 runs
// the SOR pass at compile-time bound sor_k (the largest of the table), voxel > 0 the voxel pass.
cudaError_t launch_cloud_post(float4* xyzi, uint32_t* point_counts, uint32_t n_scans, uint32_t stride,
                              uint32_t sor_k, float sor_alpha, float voxel, const CloudWorkspace& ws,
                              const uint32_t* list, const uint32_t* list_count, cudaStream_t stream, int* launched,
                              const CloudTable& tab = CloudTable{});
// fuse + all-gather through peer memory (NVLink P2P, CUDA IPC)
constexpr uint32_t kMaxPeers = 16;
constexpr uint32_t kPeerHeaderBytes = 256;
struct PeerBases {
  unsigned char* base[kMaxPeers];
};
cudaError_t launch_cloud_fuse_push(const float4* xyzi, const uint32_t* point_counts, uint32_t n_scans,
                                   uint32_t stride, const PeerBases& peers, uint32_t world, uint32_t rank,
                                   uint32_t slot_points, uint32_t* offsets, uint32_t* total, cudaStream_t stream,
                                   int* launched);
// capacity: points `fused` can hold (points past it are dropped; *total still reports the true count)
cudaError_t launch_cloud_fuse(const float4* xyzi, const uint32_t* point_counts, uint32_t n_scans,
                              uint32_t stride, float4* fused, uint32_t capacity, uint32_t* offsets, uint32_t* total,
                              cudaStream_t stream, int* launched);

}  // namespace rpl
