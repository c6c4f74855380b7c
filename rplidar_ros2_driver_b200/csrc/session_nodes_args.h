// session_nodes_args.h -- argument blocks of the session nodes kernels (session_nodes.cu): the directory of the
// packed grabbed-node buffers of a stream session's last push, and the gather of the buffers that are not ascended.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {

// One CTA over every slot of the push.  Slot i's buffer holds views[i].y nodes and starts at offsets[i], the exclusive
// scan in slot order of the counts rounded up to even; *total is the end of the last buffer.  When *total exceeds
// `capacity` every count is reported as 0 and no buffer is placed.
struct NodeDirArgs {
  const uint2* views;           // [n_slots] {first, count} of the push's scans
  uint32_t n_slots, max_scans;
  uint32_t chunk_slots;         // slots per chunk of the push (its views count from their chunk's first stream)
  uint32_t rebase;              // != 0: place[] counts from the first buffer of the slot's chunk (one chunk per block)
  const uint8_t* ascend;        // [n_slots / max_scans] nullable: the streams whose buffers are ascended
  uint32_t ascend_all;          // ascend == nullptr: every stream's are (!= 0) or none is
  unsigned long long capacity;  // nodes
  unsigned long long* offsets;  // [n_slots] out
  uint32_t* counts;             // [n_slots] out
  uint32_t* status;             // [n_slots] out: RPL_RESULT_OK for the slots the scan kernels do not serve
  unsigned long long* total;    // [1] out
  // [n_slots] out, ScanBatchArgs::out_first of the scan kernels: the buffer's position for an ascended slot; position
  // | kOutSkip for a slot the gather copies; all ones for a slot without a buffer (unused, or over capacity)
  unsigned long long* place;
};
cudaError_t launch_node_directory(const NodeDirArgs& a, cudaStream_t stream);

// copies the scans of slots [0, n_slots) whose place[] says so from their views to out + position
struct NodeGatherArgs {
  const uint2* nodes;  // the chunk's first stream's arena region (16-byte aligned)
  const uint2* views;  // [n_slots]
  const unsigned long long* place;
  uint32_t n_slots;
  uint2* out;          // 16-byte aligned; positions are even
};
cudaError_t launch_node_gather(const NodeGatherArgs& a, int num_sms, cudaStream_t stream);

}  // namespace rpl
