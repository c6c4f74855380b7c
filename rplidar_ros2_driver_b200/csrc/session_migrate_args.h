// session_migrate_args.h -- the stream record of rpl_capsule_stream_export / _import (session_migrate.cu): one stream's
// carried state, as plain little-endian bytes, and the argument block of the kernels that pack and unpack it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "decode_args.h"

namespace rpl {

// A record, every part 16-byte aligned within it (records start 16-byte aligned):
//   [0, 32)    header, uint32 words kRec*: magic, version, kind (0 framed, 1 byte session), answer type, max_nodes,
//              L (nodes of the open revolution), stamp flags (kRecOpenKnown, kRecRxKnown), 0
//   [32, 224)  the held record (kHeldWords words)
//   then, for a capsule answer type in a byte session, the framer record (kFramerWords words)
//   then the open revolution's scan-begin stamp and the held capsule's receive time (uint64 each; 0 where not known),
//   the 14 uint64 counters, and the L open nodes (8 bytes each), oldest first.
constexpr uint32_t kRecMagic = 0x4D4C5052u;  // "RPLM"
constexpr uint32_t kRecVersion = 1;
constexpr uint32_t kRecWordMagic = 0, kRecWordVersion = 1, kRecWordKind = 2, kRecWordType = 3, kRecWordMaxNodes = 4,
                   kRecWordOpen = 5, kRecWordFlags = 6, kRecWordReserved = 7;
constexpr uint32_t kRecOpenKnown = 1u, kRecRxKnown = 2u;
constexpr uint32_t kRecHeaderBytes = 32, kRecHeldBytes = 4 * kHeldWords, kRecFramerBytes = 4 * kFramerWords;
constexpr uint32_t kRecStampBytes = 16, kRecCounterBytes = sizeof(StreamCounters);

// the record's fixed part in front of its nodes, with or without a framer record
__host__ __device__ constexpr uint32_t record_fixed_bytes(bool framer) {
  return kRecHeaderBytes + kRecHeldBytes + (framer ? kRecFramerBytes : 0u) + kRecStampBytes + kRecCounterBytes;
}
static_assert(record_fixed_bytes(false) % 16 == 0 && record_fixed_bytes(true) % 16 == 0 && kRecHeldBytes % 16 == 0 &&
                  kRecFramerBytes % 16 == 0 && kRecCounterBytes % 16 == 0,
              "every part of a record stays 16-byte aligned");

// Records [0, n) at records + offsets[i] (16-byte aligned), record i being stream streams[i] of the session.  The
// session's arrays are those its next push reads: arena, carry_len and open_ts of arena `parity`.
struct MigrateArgs {
  uint8_t* records;
  const unsigned long long* offsets;  // [n]
  const uint32_t* streams;            // [n]
  uint32_t n;
  uint2* arena;                       // [n_streams][stride_nodes]: the open revolution right-aligned in the first
  uint32_t stride_nodes, max_nodes;   // max_nodes slots
  uint32_t* carry_len;                // [n_streams]
  unsigned long long* open_ts;        // [n_streams]
  unsigned long long* held_rx;        // [n_streams]
  uint32_t* held;                     // [n_streams][kHeldWords]
  uint32_t* framer;                   // [n_streams][kFramerWords] (a capsule byte session's, else nullptr)
  StreamCounters* counters;           // [n_streams]
  // pack only: the header's kind, each record's answer type ([n]), and whether the session's stamps are kept (0: its
  // last push was unstamped, so no stream knows its stamps)
  uint32_t kind;
  const uint32_t* types;
  uint32_t stamps_known;
};
// one CTA per record at a time over a grid of at most num_sms * 8
cudaError_t launch_stream_pack(const MigrateArgs& a, int num_sms, cudaStream_t stream);
cudaError_t launch_stream_unpack(const MigrateArgs& a, int num_sms, cudaStream_t stream);

}  // namespace rpl
