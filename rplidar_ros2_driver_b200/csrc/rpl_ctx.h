// rpl_ctx.h -- the context object behind the C-ABI (include/rpl_b200.h), shared by the translation units
// that implement entry points (rpl_capi.cu, exchange.cu).  Internal: not part of the boundary.
#pragma once
#include <cuda_runtime.h>

#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rpl_b200.h"
#include "cloud_args.h"
#include "scan_args.h"

constexpr int kLanes = 2;  // host-buffer pipeline depth (copy/compute overlap; three lanes measured slower: 4.8 vs 5.6 Gpoints/s)

struct Lane {
  cudaStream_t stream = nullptr;
  uint32_t* fallback_list = nullptr;
  uint32_t* fallback_count = nullptr;
  rpl::FastWorkspace fws{};
  rpl::GeneralWorkspace gws{};
  rpl::CloudWorkspace cws{};   // lane 0 owns the tables and the post-pass scratch; the others alias its tables
  bool owns_cws = false;
  // The scan scratch above (fallback list and count, fws, gws; lane 0's also the post-pass cws) serves one call's
  // kernels at a time, whatever stream the call runs on: each section that uses it waits on this event first and
  // records it after its last reader (scratch_enter / scratch_leave in rpl_capi.cu).
  cudaEvent_t scratch_free = nullptr;
  // device staging of every host-buffer call (batches, the chain, the sessions' host pushes, the single-stream
  // decoders): one block, grown before a call's chunk loop, that each call carves into the regions of one chunk
  unsigned char* stage = nullptr;
  size_t stage_bytes = 0;
};

struct rpl_ctx {
  int device = 0;
  uint32_t max_nodes = 0, max_scans = 0;
  int num_sms = 0;
  int fast_grid = 0, tma_grid[3] = {0, 0, 0}, general_grid = 0;  // tma_grid by scan_tma mode (B, A, cloud)
  int tma_clusters = 0;  // resident two-CTA clusters of scan_tma_cluster_kernel
  Lane lane[kLanes];
  std::string err;
  uint64_t launches = 0;
  // pinned mirrors of the small per-scan arrays of the host-buffer calls: keeps every copy of
  // the pipeline asynchronous even when the caller's small arrays are pageable
  uint32_t* h_counts = nullptr;
  uint32_t* h_small = nullptr;  // [4][max_scans]: beams, angle_increment bits, status, path
  // single-scan fast lane (rpl_scan / rpl_ascend_scan / rpl_laserscan): one pinned host block
  // and one device block laid out [nodes in][small][nodes out][ranges][intensities] so that a
  // scan costs one H2D copy, one or two kernel launches and one D2H copy
  unsigned char* h_one = nullptr;
  unsigned char* d_one = nullptr;
  size_t one_stride = 0;  // max_nodes rounded up to even
  // scratch of rpl_assemble_scans_dev (grown on demand)
  uint32_t* d_reset_prefix = nullptr;
  uint2* d_desc = nullptr;
  size_t reset_prefix_cap = 0, desc_cap = 0;
  cudaEvent_t asm_done = nullptr;   // the wire-to-LaserScan chunks of every lane and stream share the assemble scratch
  bool profile = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_fast, prof_general;
};

inline bool cuda_ok(rpl_ctx* c, cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  char buf[256];
  std::snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  c->err = buf;
  return false;
}
#define RPL_CUDA(c, call, code)                   \
  do {                                            \
    if (!cuda_ok((c), (call), #call)) return (code); \
  } while (0)

// Selects the context's device for an entry point and resolves the stream it runs on: the caller's, or the
// context's default stream (lane 0) when none is given.
inline bool enter_device(rpl_ctx* c, void* stream, cudaStream_t* st) {
  *st = stream ? static_cast<cudaStream_t>(stream) : c->lane[0].stream;
  return cuda_ok(c, cudaSetDevice(c->device), "cudaSetDevice(c->device)");
}

// device buffers of 8-byte records (nodes, 64-bit stamps) are accessed with 8-byte loads and stores
inline bool misaligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) != 0; }
