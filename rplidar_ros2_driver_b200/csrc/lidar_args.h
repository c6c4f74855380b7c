// lidar_args.h -- one lidar's settings, as the decode, assembly, scan and message kernels read them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {

struct TimingDesc {  // sl::SlamtecLidarTimingDesc without the bool
  uint32_t sample_duration_us, native_baudrate, linkage_delay_us, native_interface_type;
};

// rpl_lidar_settings, byte for byte: a stream session's per-stream table (rpl_*_stream_set_lidars), read by the calls
// that pass RPL_FLAG_PER_STREAM / RPL_CLOUD_PER_STREAM instead of their own params and timing
struct LidarSettings {
  uint8_t is_new_protocol, mode_a, inverted, pad;
  TimingDesc timing;
};

// How a stream's cloud runs in a call with RPL_CLOUD_PER_STREAM_CHAIN: no cloud; window + xyz only; SOR / voxel grid
// that the shared-memory kernel can fuse (its 32-bit cell keys and accumulators are exact); SOR / voxel grid as the
// separate passes
enum CloudRoute : uint8_t { kCloudOff, kCloudWindow, kCloudFused, kCloudSeparate };

// A stream's chain (rpl_capsule_stream_set_clouds) as the flagged cloud calls read it: rpl_cloud_settings's layout,
// range_max resolved against the stream's set_frames range_max, and its CloudRoute in place of `enabled`
struct CloudSettings {
  float range_min, range_max, intensity_min, voxel;
  uint32_t sor_k;
  float sor_alpha;
  uint8_t route, pad[3];
};

// a stream's route in a call whose shared-memory cloud launches are `launches` (bit 0: the window-only kernel, bit 1:
// the kernel with SOR / voxel grid fused): without the fused launch a fusable stream takes the separate passes
__host__ __device__ __forceinline__ uint32_t cloud_route(const CloudSettings& c, uint32_t launches) {
  return c.route == kCloudFused && (launches & 2u) == 0 ? (uint32_t)kCloudSeparate : (uint32_t)c.route;
}

}  // namespace rpl
