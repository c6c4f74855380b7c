// delay_model.cuh -- the SDK's per-sample delay model, shared by the timestamp kernels (timestamps.cu) and the stamped
// stream-session assembler (assemble.cu).
//
// A node's stamp is "receive time of a capsule minus a delay" (reference src/sdk/src/dataunpacker/unpacker/:
// _getSampleDelayOffsetInLegacyMode handler_normalnode.cpp:49-68, ...InExpressMode handler_capsules.cpp:55-76,
// ...InHQMode handler_hqnode.cpp:53-72, ...InUltraBoostMode handler_capsules.cpp:272-293, ...InDenseMode :586-607,
// ...InUltraDenseMode :795-816).  For the node at position pos of the capsule released by capsule j:
//   stamp = rx(prev_base ? j - 1 : j) - base - (group >= 0 ? (group - pos) * sd : 0).
#pragma once
#include "decode_args.h"

namespace rpl {

// internal linkage, as when it lived in timestamps.cu alone: the kernels that take a DelayModel keep their names
namespace {

struct DelayModel {
  unsigned long long base;  // filter + half sample + transmission + linkage
  unsigned long long sd;    // sample duration
  int group;                // last sample index of a capsule (-1: no grouping delay)
  uint32_t per;             // nodes per capsule
  bool prev_base;           // stamps count from the previous capsule's rx time (express, ultra)
};

__host__ __device__ inline DelayModel delay_model(uint32_t ans, TimingDesc t) {
  unsigned long long def_baud = 115200, size = 5;
  DelayModel m{};
  m.group = -1;
  m.per = 1;
  switch (ans) {
    case 0x81: break;
    case 0x82: size = 84; m.group = 31; m.per = 32; m.prev_base = true; break;
    case 0x83: def_baud = 1000000; size = 8; m.per = 96; break;
    case 0x84: def_baud = 256000; size = 132; m.group = 95; m.per = 96; m.prev_base = true; break;
    case 0x85: def_baud = 256000; size = 84; m.group = 39; m.per = 40; break;
    default: def_baud = 1000000; size = 170; m.group = 63; m.per = 64; break;  // 0x86
  }
  const unsigned long long baud = t.native_baudrate ? t.native_baudrate : def_baud;
  unsigned long long tx = 1000000ull * size * 10ull / baud;
  if (t.native_interface_type == 1u) tx = 100;  // LIDAR_INTERFACE_ETHERNET
  m.sd = t.sample_duration_us;
  m.base = m.sd + (m.sd >> 1) + tx + t.linkage_delay_us;
  return m;
}

}  // namespace

}  // namespace rpl
