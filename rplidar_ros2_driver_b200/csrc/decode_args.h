// decode_args.h -- argument blocks of the decode, framing, timestamp and assembly kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "lidar_args.h"

namespace rpl {

// A mixed byte session's launch over the streams of one answer type (rpl_capsule_stream_create_bytes_mixed): the
// framer, decoder and assembler take their regions as for the whole chunk, n_streams is the length of the list, and CTA
// slot i serves stream streams[i] of the chunk.  capsule_stride: bytes per stream of the framed capsules (the framer's
// output, the capsule decoder's input), which every answer type's slots share.
struct StreamList {
  const uint32_t* streams;  // [n_streams] chunk-relative stream indices, device
  uint32_t capsule_stride;
};

// the capsule formats (decode_formats.cu): 0x82 express, 0x83 HQ, 0x84 ultra, 0x85 dense, 0x86 ultra-dense
struct CapsuleDecodeArgs {
  const uint8_t* capsules;        // [n_streams][stride_capsules][capsule bytes]
  const uint32_t* counts;         // [n_streams]
  uint32_t n_streams, stride_capsules;
  uint32_t sample_duration_us;    // SlamtecLidarTimingDesc::sample_duration_uS (jump threshold)
  // words per stream of state_in / state_out: 1 = {last node sync bit} (the dense entry points), 2 = {last node
  // sync bit, last distance} (rpl_decode_capsules_batch_dev)
  uint32_t state_words;
  const uint32_t* state_in;       // [n_streams][state_words] (nullable: 0)
  uint2* nodes_out;               // [n_streams][stride_capsules * nodes per capsule]
  uint32_t* node_counts;          // [n_streams]
  uint32_t* capsule_status;       // nullable
  uint32_t* capsule_node_offset;  // nullable
  uint32_t* state_out;            // [n_streams][state_words] nullable
  // positions (node offsets) of the scan-start nodes of every stream, in no particular order (nullable; the dense
  // entry points only): what rpl_assemble_scan_views_dev otherwise finds by reading every node again
  uint32_t* scan_starts;          // [n_streams][starts_stride]
  uint32_t* scan_start_counts;    // [n_streams] (may exceed starts_stride: the list is then incomplete)
  uint32_t starts_stride;
  // stream session only (node_stride != 0, any capsule format): the nodes go to nodes_out + s * node_stride +
  // node_first (behind the session's carry slots) instead of nodes_out + s * stride_capsules * nodes per capsule, and
  // counts above stride_capsules are clamped to it.  Every format but HQ besides lets the capsule each stream held
  // back at the end of the previous push enter as the predecessor of its first capsule; state_in / state_out are
  // unused then: the decoder's cross-capsule state travels in the held record.
  uint32_t* held;                 // [n_streams][kHeldWords], read and rewritten in place (HQ: unused)
  uint32_t node_stride, node_first;
  // stream session only, nullable: each stream's jump threshold from its own entry's sample duration instead of
  // sample_duration_us
  const LidarSettings* lidars;    // [n_streams]
};

// a held-capsule record, sized for the largest capsule (ultra-dense, 170 bytes): words 0..42 the capsule's bytes,
// 43 its frame and checksum held (1) or not (0), 44 its start angle (q8), 45 the last released node's scan-start flag
// (dense, ultra-dense), 46 the smoothed last distance (ultra-dense's _last_dist_q2).  All zero: nothing held, a fresh
// stream.  The standard-node session (0x81) uses the same record for its byte machine: word 0 the last four bytes of
// the stream so far (oldest in the low byte), 43 the machine's state (bytes of the unfinished record, 0..4).
constexpr uint32_t kHeldCapsuleWords = 43, kHeldOk = 43, kHeldStart = 44, kHeldSync = 45, kHeldLast = 46,
                   kHeldWords = 48;

// a stream session's counters of one stream (rpl_stream_counters byte for byte), accumulated by the kernels of every
// push: the framer or the 0x81 decoder count the bytes, the assembler the capsule reports and the holder's losses
struct StreamCounters {
  unsigned long long bytes_in, frames, skipped_bytes, bad_frames, checksum_errors, encoder_resets, scan_resets,
      discarded_capsules, nodes, nodes_unopened, nodes_overwritten, scans_rewound, scans_published, scans_unreturned;
};

// 5-byte standard nodes from raw byte streams
struct NormalDecodeArgs {
  const uint8_t* bytes;           // [n_streams][stride_bytes]
  const uint32_t* byte_counts;    // [n_streams]
  uint32_t n_streams, stride_bytes;
  uint2* nodes_out;               // [n_streams][stride_bytes / 5]
  uint32_t* node_counts;          // [n_streams]
  uint32_t* fsm_state_out;        // [n_streams] nullable: bytes buffered when the stream ended
  uint32_t* node_end;             // [n_streams][stride_bytes / 5] nullable: index of each record's last byte
  // stream session only (node_stride != 0): the nodes go to nodes_out + s * node_stride + node_first (behind the
  // session's carry slots), counts above stride_bytes are clamped to it, and the stream enters in the state and with
  // the last four bytes its held record keeps (written back at the end); fsm_state_out is unused then, and node_end
  // (nullable, [n_streams][node_stride - node_first]) is written for the scan-start records only
  uint32_t* held;                 // [n_streams][kHeldWords], read and rewritten in place
  uint32_t node_stride, node_first;
  // stream session only: each stream's counters, given bytes_in, frames (records) and skipped_bytes
  StreamCounters* counters;       // [n_streams]
};

// per-sample timestamps (timestamps.cu; TimingDesc: lidar_args.h)
struct TimestampArgs {
  const unsigned long long* capsule_rx_us;  // [n_streams][stride_capsules]
  const uint32_t* capsule_status;
  const uint32_t* capsule_node_offset;
  const uint32_t* capsule_counts;           // [n_streams]
  uint32_t n_streams, stride_capsules;
  unsigned long long* node_ts_us;           // [n_streams][stride_capsules * nodes per capsule]
};
struct NormalTimestampArgs {
  const uint32_t* node_end;                 // [n_streams][stride_nodes] (decode_normal's report)
  const uint32_t* node_counts;              // [n_streams]
  uint32_t n_streams, stride_nodes, chunk_bytes, stride_chunks;
  const unsigned long long* chunk_rx_us;    // [n_streams][stride_chunks]
  unsigned long long* node_ts_us;           // [n_streams][stride_nodes]
};
cudaError_t launch_node_timestamps(uint32_t ans_type, const TimingDesc& t, const TimestampArgs& a, cudaStream_t stream);
cudaError_t launch_normal_timestamps(const TimingDesc& t, const NormalTimestampArgs& a, cudaStream_t stream);

// list (nullable): a mixed byte session's streams of this answer type (stream session instantiations only)
cudaError_t launch_decode_capsules(uint32_t ans_type, const CapsuleDecodeArgs& a, int grid, cudaStream_t stream,
                                   const StreamList* list = nullptr);
cudaError_t launch_decode_normal(const NormalDecodeArgs& a, int grid, cudaStream_t stream,
                                 const StreamList* list = nullptr);
cudaError_t decode_formats_configure();

struct AssembleArgs {
  const uint2* nodes;                 // [n_streams][stride_nodes] decoded node streams
  const uint32_t* node_counts;        // [n_streams]
  uint32_t n_streams, stride_nodes;
  const uint32_t* capsule_status;     // [n_streams][stride_capsules] (nullable: no scan resets)
  const uint32_t* capsule_node_offset;
  const uint32_t* capsule_counts;     // [n_streams]
  uint32_t stride_capsules;
  uint32_t max_nodes;                 // ScanDataHolder capacity (8192 in the SDK)
  uint32_t max_scans, scan_stride;
  uint2* scans_out;                   // [n_streams][max_scans][scan_stride] (copy mode)
  uint2* views_out;                   // [n_streams][max_scans] {first node in the whole buffer, count} (view mode)
  uint2* nodes_mut;                   // view mode: the node buffer, writable (capacity rule applied in place)
  uint32_t* scan_len;                 // [n_streams][max_scans]
  uint32_t* scans_per_stream;         // [n_streams] published scans (may exceed max_scans)
  const unsigned long long* node_ts_us;  // [n_streams][stride_nodes] nullable
  unsigned long long* scan_begin_ts_us;  // [n_streams][max_scans] nullable
  const uint32_t* scan_starts;        // nullable: the decoder's list of scan-start node positions per stream
  const uint32_t* scan_start_counts;
  uint32_t starts_stride;
  uint32_t* reset_prefix;             // scratch [n_streams][stride_capsules]
  uint2* desc;                        // scratch [n_streams][max_scans]
  // stream session only (view mode, carry_len != nullptr): each stream's region of `nodes` is
  // [max_nodes carry slots][new nodes]; the first carry_len[s] nodes in front of the new ones are the revolution left
  // open by the previous push.  The revolution this call leaves open goes, capped, right-aligned into the carry slots
  // of carry_out (the other arena: the scans closed here still read this one's), its length into carry_len_out.
  const uint32_t* carry_len;          // [n_streams]
  uint2* carry_out;                   // [n_streams][stride_nodes]
  uint32_t* carry_len_out;            // [n_streams]
  // stream session only: each stream's counters, given the capsule reports' events, nodes and the holder's counters
  // (and, when counted_capsule_bytes != 0 -- a framed session's push --, frames and bytes_in: capsules x that size)
  StreamCounters* counters;           // [n_streams]
  uint32_t counted_capsule_bytes;
};

// a stamped stream-session push (launch_assemble_stamped; AssembleArgs::scan_begin_ts_us is the output, every slot
// written, unused ones 0): the stamp of each published scan's scan-start node, from the receive times of this push,
// without a per-node stamp array.  Capsule formats read AssembleArgs' capsule report, 0x81 reads node_end.
constexpr unsigned long long kRxUnknown = ~0ull;  // held_rx: the held capsule came in a push without receive times
struct AssembleStampArgs {
  uint32_t ans_type;
  TimingDesc timing;
  const unsigned long long* capsule_rx_us;  // capsule formats: [n_streams][AssembleArgs::stride_capsules]
  // 0x81: [n_streams][stride_ends], at the new-node index of every scan-start record the push-relative index of its
  // last byte (decode_normal's stamped instantiation; other entries undefined); chunk c covers bytes
  // [c * chunk_bytes, (c + 1) * chunk_bytes) of the push
  const uint32_t* node_end;
  uint32_t stride_ends, chunk_bytes, stride_chunks;
  const unsigned long long* chunk_rx_us;    // 0x81: [n_streams][stride_chunks]
  // the stamp of the open revolution entering and leaving the push, beside carry_len (0: unknown)
  const unsigned long long* open_ts_in;     // [n_streams]
  unsigned long long* open_ts_out;          // [n_streams]
  // express, ultra: receive time of the held capsule, read and rewritten in place (kRxUnknown: never given)
  unsigned long long* held_rx;              // [n_streams]
  // 0: the previous push had no receive times, so open_ts_in and held_rx are stale and count as unknown
  uint32_t prev_stamped;
  // the session's own copy of every slot's scan-begin stamp, and its end stamp: the stamp of the scan-start node that
  // closed the scan, which opens the next scan whether that one is published, dropped past max_scans or reset
  unsigned long long* slot_begin_us;        // [n_streams][AssembleArgs::max_scans], unused slots 0
  unsigned long long* slot_end_us;          // [n_streams][AssembleArgs::max_scans], unused slots 0
  // nullable: each stream's delay model from its own entry's timing instead of `timing`
  const LidarSettings* lidars;              // [n_streams]
};

// byte-level framing with the SDK's resynchronisation (frame.cu)
struct FrameArgs {
  const uint8_t* bytes;           // [n_streams][stride_bytes] raw capsule streams
  const uint32_t* byte_counts;    // [n_streams]
  uint32_t n_streams, stride_bytes;
  uint32_t capsule_bytes;         // frame size of the answer type
  uint8_t* capsules_out;          // [n_streams][stride_capsules][capsule_bytes]
  uint32_t stride_capsules;
  uint32_t* capsule_counts_out;   // [n_streams]
  uint32_t* bytes_left_out;       // [n_streams] nullable: bytes of an unfinished frame at the end
};
// a byte session's framer record per stream: word kFramerPos the search position (0 waiting for byte 0, 1 waiting for
// byte 1 -- HQ: collecting --, k >= 2 collecting), which is also the number of bytes of the unfinished frame held from
// kFramerBytes on (up to the frame size - 1: 780 for HQ); kFramerLost 1 while skipped bytes wait for the next frame to
// be reported as the all-zero capsule in front of it.  All zero: a fresh stream.
constexpr uint32_t kFramerPos = 0, kFramerLost = 1, kFramerBytes = 2, kFramerWords = 200;
// the session instantiation's own arguments (FrameArgs::stride_capsules then counts capsule slots, byte counts above
// stride_bytes are clamped to it, and bytes_left_out is unused)
struct FrameStreamArgs {
  uint32_t* framer;                         // [n_streams][kFramerWords], read and rewritten in place
  // nullable: chunk c the receive time of bytes [c * chunk_bytes, (c + 1) * chunk_bytes) of the push
  const unsigned long long* chunk_rx_us;    // [n_streams][stride_chunks]
  uint32_t chunk_bytes, stride_chunks;
  unsigned long long* capsule_rx_out;       // [n_streams][stride_capsules] with chunk_rx_us: each capsule's
  StreamCounters* counters;                 // [n_streams]: given bytes_in, frames and skipped_bytes
};
cudaError_t launch_frame_capsules(const FrameArgs& a, int grid, cudaStream_t stream);
cudaError_t launch_frame_capsules_stream(const FrameArgs& a, const FrameStreamArgs& f, int grid, cudaStream_t stream,
                                         const StreamList* list = nullptr);
cudaError_t launch_assemble(const AssembleArgs& a, int grid, cudaStream_t stream, const StreamList* list = nullptr);
cudaError_t launch_assemble_stamped(const AssembleArgs& a, const AssembleStampArgs& t, int grid, cudaStream_t stream,
                                    const StreamList* list = nullptr);

}  // namespace rpl
