// lidar_args.h -- one lidar's settings, as the decode, assembly, scan and message kernels read them.
#pragma once
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

}  // namespace rpl
