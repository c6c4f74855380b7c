// cdr_args.h -- argument blocks of the CDR serialisation kernels (cdr.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "lidar_args.h"

namespace rpl {

struct LaserScanMeta {  // == rpl_laserscan_meta
  int32_t stamp_sec;
  uint32_t stamp_nanosec;
  float angle_min, angle_max, angle_increment, time_increment, scan_time, range_min, range_max;
};

// fixed part of a message, built on the host (rpl_capi.cu): copied, then patched per message
struct CdrTemplate {
  uint8_t prefix[512];
  uint32_t prefix_bytes;    // multiple of 4
  uint32_t patch_width;     // PointCloud2: offset of `width`
  uint32_t patch_row_step;  // PointCloud2: offset of `row_step`
};

struct LaserScanCdrArgs {
  const LaserScanMeta* meta;      // [n_scans] device
  const float* angle_increment;   // [n_scans] device, nullable: overrides meta[s].angle_increment
  const float* ranges;            // [n_scans][stride]
  const float* intensities;       // [n_scans][stride]
  const uint32_t* beam_counts;    // [n_scans]
  uint32_t n_scans, stride;
  uint8_t* cdr_out;               // [n_scans][cdr_stride], cdr_stride % 4 == 0
  uint32_t cdr_stride;
  uint32_t* cdr_sizes;            // [n_scans] nullable
};

struct PointCloudCdrArgs {
  const uint32_t* stamps;         // [n_clouds][2] {sec, nanosec}
  const float* xyzi;              // [n_clouds][stride][4]
  const uint32_t* point_counts;   // [n_clouds]
  uint32_t n_clouds, stride;
  uint8_t* cdr_out;               // [n_clouds][cdr_stride], cdr_stride % 16 == 0
  uint32_t cdr_stride;
  uint32_t* cdr_sizes;
};

cudaError_t launch_laserscan_cdr(const LaserScanCdrArgs& a, const CdrTemplate& t, cudaStream_t stream);
cudaError_t launch_pointcloud2_cdr(const PointCloudCdrArgs& a, const CdrTemplate& t, cudaStream_t stream);

// ---- packed messages of a stream session's last push (rpl_*_stream_{laserscan,cloud}_msgs*) ----------------------
// One stream's message settings, built on the host by rpl_*_stream_set_frames: the bytes every message of the stream
// starts with -- encapsulation header, stamp (zero here, patched per message), frame_id string padded to 4.
constexpr uint32_t kMsgHeaderWords = 70;  // 4 + 8 + 4 + 256 (frame_id <= 255 characters + NUL) bytes, rounded up
struct StreamMsgHeader {
  uint32_t bytes;                  // multiple of 4
  float range_max;                 // LaserScan range_max
  uint32_t w[kMsgHeaderWords];
};

// The PointCloud2 members between the header and the data (height .. data length): identical bytes for every frame
// id, since the header ends 4-aligned and nothing behind it is aligned to more than 4
struct CloudTail {
  uint32_t w[29];
  uint32_t bytes;                          // 116
  uint32_t at_width, at_row_step, at_data;  // word indices patched per message
};

// kScanCloud: the projection of each slot's LaserScan (scan_cloud.cu), a PointCloud2 of point_step-byte records;
// kRescan: the LaserScan re-gridded from that projection (rescan.cu), of its stream's fixed beam count
enum class MsgKind : uint32_t { kLaserScan, kPointCloud2, kScanCloud, kRescan };

// sizes and offsets pass: one CTA over every slot
struct MsgTableArgs {
  MsgKind kind;
  const StreamMsgHeader* hdr;      // [n_slots / max_scans]
  const uint32_t* counts;          // [n_slots] beams / points
  const uint2* views;              // [n_slots] PointCloud2: a slot has a message iff its view count is > 0
  uint32_t n_slots, max_scans;
  unsigned long long capacity;
  unsigned long long* offsets;     // [n_slots] out: exclusive scan of the sizes rounded up to 16
  uint32_t* sizes;                 // [n_slots] out: message bytes, 0 for no message or when the total exceeds capacity
  unsigned long long* total;       // out: end of the last message
  const CloudSettings* clouds;     // [n_slots / max_scans] nullable, PointCloud2: a kCloudOff stream's slots have none
  // kScanCloud: a slot has a message iff its LaserScan has beams (beams[i] > 0), of header + tail_bytes + point_step *
  // counts[i] + 1 (is_dense) bytes
  const uint32_t* beams;
  uint32_t tail_bytes, point_step;
  // kRescan (counts: the LaserScans' beams): a slot has a message iff its LaserScan has beams and its stream's bins[s]
  // (the entry's ranges_size, 0 for a disabled entry) is > 0, of header + 36 + 4 * bins[s] bytes
  const uint32_t* bins;
};

// the writers, over slots [slot0, slot0 + n) (slot indices count from the first slot of the call)
struct MsgWriteArgs {
  const StreamMsgHeader* hdr;
  const unsigned long long *begin_us, *end_us;  // [n_slots] nullable together: an unstamped push (stamps 0)
  long long clock_offset_ns;
  const uint32_t* counts;          // [n_slots]
  const float *ranges, *intensities, *angle_increment;  // LaserScan: [n_slots][stride], [n_slots]
  const float* xyzi;               // PointCloud2: [n_slots][stride][4]
  uint32_t stride, max_scans, mode_a;
  uint32_t slot0, n;
  const unsigned long long* offsets;
  const uint32_t* sizes;
  uint8_t* out;                    // message i at out + offsets[i] - out_base
  unsigned long long out_base;
  const LidarSettings* lidars;     // [n_slots / max_scans] nullable: LaserScan slot i takes its stream's mode, not mode_a
};

cudaError_t launch_msg_table(const MsgTableArgs& a, cudaStream_t stream);
cudaError_t launch_laserscan_msgs(const MsgWriteArgs& a, uint32_t max_beams, cudaStream_t stream);

// ---- messages written by a push (rpl_capsule_stream_push_{laserscan,cloud}_msgs*) -------------------------------
// The directory of one chunk of the push, one CTA, every pointer at the chunk's first slot (stream).  A published slot
// (k < min(scans_per_stream[s], max_scans)) takes, rounded up to 16, its LaserScan message at the view's node count (a
// bound, known before the scan kernels run) or its PointCloud2 message at the cloud's point count (the exact size,
// known once the cloud kernels have run); an unused slot 0.  offsets[i] = *carry (the previous chunk's end; 0 for the
// push's first chunk) + the exclusive scan of the chunk's rounded sizes; the chunk's end goes back to *carry.  A slot
// whose message ends past `capacity` gets no message.
struct PushMsgDirArgs {
  const uint2* views;               // [n_slots] the chunk's scans
  const uint32_t* scans_per_stream; // [n_slots / max_scans]
  const StreamMsgHeader* hdr;       // [n_slots / max_scans]
  uint32_t n_slots, max_scans;
  uint32_t first;                   // != 0: the push's first chunk (the carry is not read)
  uint32_t rebase;                  // != 0: place[] counts from the chunk's first offset (else from 0)
  unsigned long long capacity;
  unsigned long long* carry;        // [1] in / out; PointCloud2: [2], the end of the last message in carry[1]
  unsigned long long* offsets;      // [n_slots] out
  // [n_slots] out, LaserScan, ScanBatchArgs::msg_ranges: where the message's ranges start (message position + header
  // + 32); kOutSkip for a slot without a message
  unsigned long long* place;
  unsigned long long* extent;       // [3] out, nullable: the chunk's first offset, the end of its last message that
                                    // fits, the total so far
  unsigned long long* total;        // [1] out, nullable: the total so far -- LaserScan: the end of the chunk's bounds;
                                    // PointCloud2: the end of the last message (msg_table_kernel's total)
  const uint32_t* counts;           // [n_slots] PointCloud2: the clouds' point counts
  uint32_t* sizes;                  // [n_slots] out, PointCloud2: the message's bytes when it fits, else 0
  const CloudSettings* clouds;      // [n_slots / max_scans] nullable, PointCloud2: a kCloudOff stream's slots have none
  // kScanCloud (sizes, total and carry [2] as PointCloud2): slot i has a message iff its LaserScan message was written
  // (scan_sizes[i] > 0), of header + tail_bytes + point_step * counts[i] (the kept beams) + 1 (is_dense) bytes
  const uint32_t* scan_sizes;
  uint32_t tail_bytes, point_step;
  // kRescan (sizes, total and carry [2] as PointCloud2): counts is [n_slots / max_scans], each stream's entry's
  // ranges_size (0 for a disabled entry); slot i has a message iff its LaserScan message was written (scan_sizes[i] >
  // 0) and counts[s] > 0, of header + 36 + 4 * counts[s] bytes
};
cudaError_t launch_push_msg_dir(const PushMsgDirArgs& a, MsgKind kind, cudaStream_t stream);
// The fixed part of every placed message of slots [0, a.n) once the scan kernels have written its arrays (a's hdr,
// begin_us / end_us, counts, angle_increment, lidars at the chunk's first slot; its offsets, sizes, out_base unused):
// message i at a.out + place[i] - header bytes - 32; sizes[i] its bytes, 0 for no message.
cudaError_t launch_laserscan_placed(const MsgWriteArgs& a, const unsigned long long* place, uint32_t* sizes,
                                    cudaStream_t stream);
cudaError_t launch_pointcloud2_msgs(const MsgWriteArgs& a, const CloudTail& t, uint32_t max_points, cudaStream_t stream);

}  // namespace rpl
