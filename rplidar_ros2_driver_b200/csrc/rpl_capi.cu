// rpl_capi.cu -- the C-ABI of librplidar_b200.so (include/rpl_b200.h).
//
// Host-side glue only: context, workspaces, streams, the chunked host<->device pipeline of
// the host-buffer entry points, and kernel launches.  There is no CPU implementation of the
// path in this library: every entry point either runs the CUDA kernels or fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rpl_b200.h"
#include "cloud_args.h"
#include "cloud_footprint_args.h"
#include "cdr_args.h"
#include "decode_args.h"
#include "rescan_args.h"
#include "scan_args.h"
#include "scan_cloud_args.h"
#include "scan_filter_args.h"
#include "session_migrate_args.h"
#include "session_nodes_args.h"

namespace rpl {
cudaError_t launch_synth(uint64_t first_scan_id, uint32_t n_scans, uint32_t n, uint32_t stride,
                         int variant, uint2* nodes, uint32_t* counts, cudaStream_t stream);
}

static_assert(sizeof(rpl_node_hq) == 8, "packed node must be 8 bytes");

#include "rpl_ctx.h"

namespace {

template <class P>
cudaError_t dev_alloc(P** p, size_t count) {
  return cudaMalloc(reinterpret_cast<void**>(p), std::max<size_t>(count, 1) * sizeof(P));
}

void free_lane(Lane& l) {
  cudaFree(l.fallback_list);
  cudaFree(l.fallback_count);
  cudaFree(l.fws.group);
  cudaFree(l.gws.keyf);
  cudaFree(l.gws.idx0);
  cudaFree(l.gws.idx1);
  cudaFree(l.gws.vidx);
  cudaFree(l.gws.cell);
  if (l.owns_cws) rpl::cloud_workspace_free(l.cws);
  cudaFree(l.stage);
  if (l.scratch_free) cudaEventDestroy(l.scratch_free);
  if (l.stream) cudaStreamDestroy(l.stream);
  l = Lane{};
}

// Carves consecutive 256-byte-aligned regions off a lane's staging block; with base == nullptr it only counts their
// bytes, so that one layout function both sizes the block and lays it out.  Regions lie in the order they are taken;
// a braced list is evaluated left to right, so a layout may take them all in the initializer of its Regions struct.
struct Carve {
  unsigned char* base = nullptr;
  size_t bytes = 0;
  template <class T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (count * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

// Grows the staging blocks of lanes [0, lanes) to what layout(Carve&) takes.  Called before a call's chunk loop only:
// a lane's stream is drained before its block is replaced, since an earlier call's copies may still use it.
template <class Layout>
rpl_result grow_stage(rpl_ctx* c, int lanes, Layout layout) {
  Carve k;
  layout(k);
  for (int i = 0; i < lanes; ++i) {
    Lane& l = c->lane[i];
    if (l.stage_bytes >= k.bytes) continue;
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);
    cudaFree(l.stage);
    l.stage = nullptr;
    l.stage_bytes = 0;
    RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&l.stage), k.bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
    l.stage_bytes = k.bytes;
  }
  return RPL_RESULT_OK;
}

// The kernel that runs ahead of scan_general_kernel; the general kernel then serves only the scans it hands on.
// kNone: the general kernel serves every scan.
enum class FastKernel { kNone, kSmall, kCluster, kTma, kFast };

// Sums every profiled launch queued so far into c->prof_ms / prof_n and resets the stamp records
// (rpl_ctx::prof_stamps).  Synchronises the device.
rpl_result prof_drain(rpl_ctx* c) {
  RPL_CUDA(c, cudaDeviceSynchronize(), RPL_RESULT_OPERATION_FAIL);
  std::vector<unsigned long long> st(2 * (size_t)c->prof_stamps_used);
  if (!st.empty())
    RPL_CUDA(c, cudaMemcpy(st.data(), c->prof_stamps, st.size() * 8, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  auto sum = [&](std::vector<rpl_ctx::ProfLaunch>& v, int kind) {
    for (const auto& pl : v) {
      if (pl.stamp >= 0) {
        const unsigned long long t0 = st[2 * pl.stamp], t1 = st[2 * pl.stamp + 1];
        if (t1 > t0) c->prof_ms[kind] += (double)(t1 - t0) * 1e-6;
      } else {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, pl.e0, pl.e1) == cudaSuccess) c->prof_ms[kind] += t;
        cudaEventDestroy(pl.e0);
        cudaEventDestroy(pl.e1);
      }
      c->prof_n[kind]++;
    }
    v.clear();
  };
  sum(c->prof_fast, 0);
  sum(c->prof_general, 1);
  if (c->prof_stamps_used != 0) {  // {earliest start, latest end} = {all ones, 0}
    RPL_CUDA(c, cudaMemset2D(c->prof_stamps, 16, 0xFF, 8, c->prof_stamps_used), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemset2D(c->prof_stamps + 1, 16, 0, 8, c->prof_stamps_used), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaDeviceSynchronize(), RPL_RESULT_OPERATION_FAIL);
  }
  c->prof_stamps_used = 0;
  return RPL_RESULT_OK;
}

// the stamp record of one profiled launch (nullptr with c->err set on failure)
unsigned long long* prof_take(rpl_ctx* c) {
  if (c->prof_stamps_used == rpl_ctx::kProfStamps && prof_drain(c) != RPL_RESULT_OK) return nullptr;
  return c->prof_stamps + 2 * (size_t)c->prof_stamps_used++;
}

// the kernel-selection rule of every scan entry point, batches and single scans alike
FastKernel pick_fast(const rpl::ScanBatchArgs& a, uint32_t flags) {
  // FORCE_GENERAL and status-only calls (no LaserScan, no ascended buffer) take the general kernel alone
  if ((flags & RPL_FLAG_FORCE_GENERAL) != 0 || (!a.ranges && !a.nodes_out && !a.xyzi && !a.msg_out))
    return FastKernel::kNone;
  // revolutions that fit shared memory (what a lidar delivers) have their own kernels
  if (rpl::scan_small_applies(a.stride) && (flags & RPL_FLAG_NO_SMALL) == 0) return FastKernel::kSmall;
  // above that the TMA kernels need every scan base 16-byte aligned, and the PointCloud2 payload exists in the
  // TMA kernel and the general kernel only
  const bool aligned = (reinterpret_cast<uintptr_t>(a.nodes) & 15u) == 0 && (a.stride & 1u) == 0;
  if (a.xyzi && !aligned) return FastKernel::kNone;
  // the ascended buffer and NO_TMA (LaserScan only) take scan_fast_kernel
  if (a.nodes_out || !aligned || ((flags & RPL_FLAG_NO_TMA) != 0 && !a.xyzi)) return FastKernel::kFast;
  // LaserScan Mode B scans too large for the shared-memory kernels but no larger than two SMs can stage
  if (!a.xyzi && !a.mode_a && rpl::scan_tma_cluster_applies(a.stride)) return FastKernel::kCluster;
  return FastKernel::kTma;
}

// Launches fast kernel k on `stream` (k != kNone); a.fallback_count is zero when it starts.  A PointCloud2 launch may
// fuse the SOR / voxel-grid passes of `cloud` (steps 4-5) into the shared-memory kernel: *post_fused tells.
// hand_off (scan views): above kSmallPostMaxNodes, fuse all the same with the shared memory sized for that many nodes,
// the longer views going to the general kernel like duplicate-key scans.
// ticket (nullable, zero when the kernel starts): the cluster kernel hands out scans from it (scan_tma.cu); without
// one, each cluster takes a fixed share.
rpl_result launch_fast(rpl_ctx* c, Lane& l, const rpl::ScanBatchArgs& a, FastKernel k, cudaStream_t stream,
                       const rpl_cloud_params* cloud = nullptr, bool* post_fused = nullptr, bool hand_off = false,
                       uint32_t* ticket = nullptr) {
  const int tma_grid = c->tma_grid[a.xyzi ? 2 : a.mode_a ? 1 : 0];
  const int grid = k == FastKernel::kCluster
                       ? 2 * (int)std::min<uint32_t>(a.n_scans, (uint32_t)c->tma_clusters)
                       : (int)std::min<uint32_t>(a.n_scans, (uint32_t)(k == FastKernel::kTma ? tma_grid : c->fast_grid));
  // the cluster kernel times itself (its general kernel runs chained behind it), the others between two events
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  unsigned long long* stamp = nullptr;
  if (c->profile && k == FastKernel::kCluster) {
    if (!(stamp = prof_take(c))) return RPL_RESULT_OPERATION_FAIL;
  } else if (c->profile) {
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, stream);
  }
  if (k == FastKernel::kSmall) {
    // SOR / voxel grid run inside the kernel when the 32-bit cell keys and accumulators are exact:
    // |cell index| < 32768 and voxel <= 4 m (scan_small.cu); otherwise as separate passes
    const bool fits = rpl::scan_small_post_applies(a.stride);
    if (a.xyzi && a.clouds) {  // per-stream clouds: the launches a.cloud_launches names (stream_cloud_chunk)
      RPL_CUDA(c, rpl::launch_scan_small(a, l.fws.max_nodes, 0u, 0.0f, 0.0f, c->num_sms, stream,
                                         fits ? 0u : rpl::kSmallPostMaxNodes),
               RPL_RESULT_OPERATION_FAIL);
      if (post_fused) *post_fused = (a.cloud_launches & 2u) != 0;
      c->launches += __builtin_popcount(a.cloud_launches);
      return RPL_RESULT_OK;
    }
    bool fuse = false;
    if (a.xyzi && cloud && (cloud->sor_k > 0 || cloud->voxel_size > 0.0f) && (fits || (hand_off && a.views)))
      fuse = cloud->voxel_size == 0.0f || (cloud->voxel_size <= 4.0f && a.range_max / cloud->voxel_size < 32000.0f);
    const uint32_t cap = fuse && !fits ? rpl::kSmallPostMaxNodes : 0u;
    RPL_CUDA(c, rpl::launch_scan_small(a, l.fws.max_nodes, fuse ? cloud->sor_k : 0u, fuse ? cloud->sor_alpha : 0.0f,
                                       fuse ? cloud->voxel_size : 0.0f, c->num_sms, stream, cap),
             RPL_RESULT_OPERATION_FAIL);
    if (post_fused) *post_fused = fuse;
  } else if (k == FastKernel::kCluster) {
    RPL_CUDA(c, rpl::launch_scan_tma_cluster(a, l.fws.max_nodes, grid, ticket, stamp, stream), RPL_RESULT_OPERATION_FAIL);
  } else if (k == FastKernel::kTma) {
    RPL_CUDA(c, rpl::launch_scan_tma(a, l.fws.max_nodes, grid, stream), RPL_RESULT_OPERATION_FAIL);
  } else {
    RPL_CUDA(c, rpl::launch_scan_fast(a, l.fws, grid, stream), RPL_RESULT_OPERATION_FAIL);
  }
  if (c->profile) {
    if (!stamp) cudaEventRecord(e1, stream);
    c->prof_fast.push_back({e0, e1, stamp ? (int)((stamp - c->prof_stamps) / 2) : -1});
  }
  // a per-stream LaserScan launch of the shared-memory kernels is one launch per mode present
  c->launches += k == FastKernel::kSmall && a.lidars && !a.xyzi ? __builtin_popcount(a.lidar_modes) : 1;
  return RPL_RESULT_OK;
}

// launches scan_general_kernel on `stream` over every scan (all_scans) or over the scans in a.fallback_list; it zeroes
// zero_next[0..1] (nullable) for the lane's next call.  chained: it directly follows the fast kernel that fills the list,
// and is launched as that kernel's programmatic dependent, so that its launch overlaps the fast kernel's tail.
rpl_result launch_general(rpl_ctx* c, Lane& l, const rpl::ScanBatchArgs& a, bool all_scans, cudaStream_t stream,
                          uint32_t* zero_next = nullptr, bool chained = false) {
  const int grid = (int)std::min<uint32_t>(a.n_scans, (uint32_t)c->general_grid);
  unsigned long long* stamp = nullptr;  // profiled: the kernel times itself, from the end of its wait on a chained start
  if (c->profile && !(stamp = prof_take(c))) return RPL_RESULT_OPERATION_FAIL;
  RPL_CUDA(c, rpl::launch_scan_general(a, l.gws, grid, all_scans, zero_next, chained, stamp, stream),
           RPL_RESULT_OPERATION_FAIL);
  if (c->profile) c->prof_general.push_back({nullptr, nullptr, (int)((stamp - c->prof_stamps) / 2)});
  c->launches++;
  return RPL_RESULT_OK;
}

// A lane's scan scratch (Lane::scratch_free) is taken by one section of kernels at a time: the device calls of every
// stream run on lane 0's, the host calls' chunks on their lane's.  A section starts, on its stream, after the lane's
// previous section has ended, and ends after its last kernel that reads the scratch.
rpl_result scratch_enter(rpl_ctx* c, Lane& l, cudaStream_t stream) {
  l.spare_queued = false;
  RPL_CUDA(c, cudaStreamWaitEvent(stream, l.scratch_free, 0), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}
rpl_result scratch_leave(rpl_ctx* c, Lane& l, cudaStream_t stream) {
  RPL_CUDA(c, cudaEventRecord(l.scratch_free, stream), RPL_RESULT_OPERATION_FAIL);
  // the next section, ordered behind this one, finds its hand-off counter zeroed by this section's general kernel
  if (l.spare_queued) l.spare_zeroed = true;
  l.spare_queued = false;
  return RPL_RESULT_OK;
}

// the fast kernel, then the general kernel for the scans it hands on (or for all), on `stream` with no host round trip;
// the caller holds lane l's scratch (scratch_enter) from before this call to after the last reader of its fallback list
rpl_result enqueue_args(rpl_ctx* c, Lane& l, rpl::ScanBatchArgs a, uint32_t flags, cudaStream_t stream,
                        const rpl_cloud_params* cloud = nullptr, bool* post_fused = nullptr, bool hand_off = false) {
  if (post_fused) *post_fused = false;
  if (a.nodes_out && !a.apply_ascend) {
    // no geometric correction requested: the buffer passes through unchanged
    // (reference lidar_driver_wrapper.cpp:330-337); a plain device copy, not kernel work
    RPL_CUDA(c, cudaMemcpy2DAsync(a.nodes_out, (size_t)a.stride * 8, a.nodes, (size_t)a.stride * 8,
                                  (size_t)a.stride * 8, a.n_scans, cudaMemcpyDeviceToDevice, stream),
             RPL_RESULT_OPERATION_FAIL);
    a.nodes_out = nullptr;
  }
  FastKernel k = pick_fast(a, flags);
  // per-stream settings, per-stream clouds and placed messages are read by the shared-memory kernels and the general
  // kernel only
  if ((a.lidars || a.msg_out || a.clouds) && k != FastKernel::kSmall) k = FastKernel::kNone;
  // this call's hand-off counter and scan ticket (Lane::fallback_count), and the lane's next call's pair, which the
  // general kernel zeroes
  l.count_parity ^= 1u;
  a.fallback_count = l.hand_off_count();
  const bool zeroed = l.spare_zeroed;
  l.spare_zeroed = false;
  if (k != FastKernel::kNone) {
    if (!zeroed)
      RPL_CUDA(c, cudaMemsetAsync(a.fallback_count, 0, 2 * sizeof(uint32_t), stream), RPL_RESULT_OPERATION_FAIL);
    const rpl_result r = launch_fast(c, l, a, k, stream, cloud, post_fused, hand_off, a.fallback_count + 1);
    if (r != RPL_RESULT_OK) return r;
  }
  const rpl_result r = launch_general(c, l, a, k == FastKernel::kNone, stream,
                                      l.fallback_count + 2 * (l.count_parity ^ 1u), k == FastKernel::kCluster);
  if (r == RPL_RESULT_OK) l.spare_queued = true;
  return r;
}

// the fields of a LaserScan launch that come from the parameters and the lane
rpl::ScanBatchArgs scan_args(const rpl_scan_params* p, const Lane& l) {
  rpl::ScanBatchArgs a{};
  a.fallback_list = l.fallback_list;
  a.is_new_protocol = p->is_new_protocol;
  a.mode_a = p->scan_processing;
  a.inverted = p->inverted;
  a.apply_ascend = p->apply_ascend;
  a.angle = l.cws.angle;
  return a;
}

// a session call's per-stream settings (RPL_FLAG_PER_STREAM): scan slot s of the call takes entry s / per of `at`,
// which points at the call's first stream's entry; at == nullptr: the call's params serve every scan
struct LidarTable {
  const rpl::LidarSettings* at = nullptr;
  uint32_t per = 0;    // scan slots per stream
  uint32_t modes = 0;  // bit 0: some stream of the session in Mode B, bit 1: in Mode A
};

// queue the scan kernels for one device-resident batch on `stream`
rpl_result enqueue_scan(rpl_ctx* c, Lane& l, const rpl_node_hq* nodes, const uint32_t* counts,
                        uint32_t n_scans, uint32_t stride, const rpl_scan_params* p,
                        rpl_node_hq* nodes_out, float* ranges, float* intens, uint32_t* beams,
                        float* inc, uint32_t* status, uint32_t* path, cudaStream_t stream,
                        const uint2* views = nullptr, unsigned long long nodes_total = 0, LidarTable lt = {},
                        uint8_t* msg_out = nullptr, const unsigned long long* msg_ranges = nullptr) {
  if (n_scans == 0) return RPL_RESULT_OK;
  if (!nodes || !counts || !p) {
    c->err = "null nodes/counts/params";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_scans > c->max_scans) {
    c->err = "n_scans exceeds the context's max_scans";
    return RPL_RESULT_INVALID_DATA;
  }
  if ((ranges == nullptr) != (intens == nullptr)) {
    c->err = "ranges and intensities must be given together";
    return RPL_RESULT_INVALID_DATA;
  }
  if (nodes_out && static_cast<const void*>(nodes_out) == static_cast<const void*>(nodes)) {
    c->err = "nodes_out must not alias nodes on the device path";
    return RPL_RESULT_INVALID_DATA;
  }
  if (misaligned8(nodes) || misaligned8(nodes_out)) {
    c->err = "node buffers must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  rpl::ScanBatchArgs a = scan_args(p, l);
  a.nodes = reinterpret_cast<const uint2*>(nodes);
  a.nodes_out = reinterpret_cast<uint2*>(nodes_out);
  a.counts = counts;
  a.n_scans = n_scans;
  a.stride = stride;
  a.ranges = ranges;
  a.intensities = intens;
  a.beam_counts = beams;
  a.angle_inc = inc;
  a.status = status;
  a.path = path;
  a.views = views;
  a.nodes_total = nodes_total;
  a.lidars = lt.at;
  a.lidar_scans = lt.per;
  a.lidar_modes = lt.modes;
  a.msg_out = msg_out;
  a.msg_ranges = msg_ranges;
  rpl_result r = scratch_enter(c, l, stream);
  if (r == RPL_RESULT_OK) r = enqueue_args(c, l, a, p->flags, stream);
  return r == RPL_RESULT_OK ? scratch_leave(c, l, stream) : r;
}

// Runs fn(lane, first, n) over `total` items in chunks of `chunk`, round-robin over the lanes, and waits for every
// lane.  A failure leaves the loop with copies possibly still in flight: nothing may still be writing into the
// caller's buffers when the error is reported, so every lane is drained first and the first error kept.
template <class F>
rpl_result run_chunks(rpl_ctx* c, uint32_t total, uint32_t chunk, F fn) {
  uint32_t ci = 0;
  for (uint32_t s0 = 0; s0 < total; s0 += chunk, ++ci) {
    const rpl_result r = fn(c->lane[ci % kLanes], s0, std::min(chunk, total - s0));
    if (r != RPL_RESULT_OK) {
      const std::string why = c->err;
      for (int i = 0; i < kLanes; ++i) cudaStreamSynchronize(c->lane[i].stream);
      c->err = why;
      return r;
    }
  }
  return rpl_ctx_synchronize(c);
}

// argument checks shared by several entry points
bool sample_duration_ok(rpl_ctx* c, uint32_t sample_duration_us) {
  if (sample_duration_us != 0 && sample_duration_us <= 1000000u) return true;
  c->err = "sample_duration_us must be in [1, 1000000]";
  return false;
}

// bytes per capsule of a capsule answer type; 0, with the error set, for any other type
uint32_t capsule_bytes(rpl_ctx* c, uint32_t ans_type) {
  const uint32_t b = rpl_capsule_bytes(ans_type);
  if (b == 0) c->err = "unknown answer type (capsule formats are 0x82..0x86)";
  return b;
}

bool frame_id_length_ok(rpl_ctx* c, size_t len) {
  if (len <= 255) return true;
  c->err = "frame_id longer than 255 characters";
  return false;
}

}  // namespace

extern "C" {

uint32_t rpl_abi_version(void) { return RPL_ABI_VERSION; }

rpl_result rpl_ctx_create(int device, uint32_t max_nodes, uint32_t max_scans, rpl_ctx** out) {
  if (!out || max_nodes == 0 || max_scans == 0) return RPL_RESULT_INVALID_DATA;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    // no CPU fallback by design
    return RPL_RESULT_OPERATION_NOT_SUPPORT;
  }
  rpl_ctx* c = new (std::nothrow) rpl_ctx();
  if (!c) return RPL_RESULT_INSUFFICIENT_MEMORY;
  c->device = device;
  c->max_nodes = max_nodes;
  c->max_scans = max_scans;
  auto fail = [&](rpl_result r) {
    std::fprintf(stderr, "[rpl_b200] rpl_ctx_create failed: %s\n", c->err.c_str());
    rpl_ctx_destroy(c);
    return r;
  };
  if (!cuda_ok(c, cudaSetDevice(device), "cudaSetDevice")) return fail(RPL_RESULT_OPERATION_FAIL);
  cudaDeviceProp prop{};
  if (!cuda_ok(c, cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties"))
    return fail(RPL_RESULT_OPERATION_FAIL);
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    c->err = "librplidar_b200 is built for sm_90a (H100) only";
    return fail(RPL_RESULT_OPERATION_NOT_SUPPORT);
  }
  c->num_sms = prop.multiProcessorCount;
  if (!cuda_ok(c, rpl::scan_fast_configure(), "scan_fast_configure") ||
      !cuda_ok(c, rpl::scan_tma_configure(), "scan_tma_configure") ||
      !cuda_ok(c, rpl::scan_small_configure(), "scan_small_configure") ||
      !cuda_ok(c, rpl::scan_general_configure(), "scan_general_configure") ||
      !cuda_ok(c, rpl::cloud_configure(), "cloud_configure") ||
      !cuda_ok(c, rpl::decode_formats_configure(), "decode_formats_configure"))
    return fail(RPL_RESULT_OPERATION_FAIL);
  const int occ = std::max(1, rpl::scan_fast_max_ctas_per_sm());
  c->fast_grid = c->num_sms * occ;
  for (int m = 0; m < 3; ++m) c->tma_grid[m] = c->num_sms * std::max(1, rpl::scan_tma_max_ctas_per_sm(m));
  c->tma_clusters = rpl::scan_tma_max_clusters();
  if (c->tma_clusters < 1) {
    c->err = "scan_tma_cluster_kernel: no two-CTA cluster fits the device";
    return fail(RPL_RESULT_OPERATION_FAIL);
  }
  c->general_grid = c->num_sms;

  for (int i = 0; i < kLanes; ++i) {
    Lane& l = c->lane[i];
    const rpl_result oom = RPL_RESULT_INSUFFICIENT_MEMORY;
    if (!cuda_ok(c, cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking), "cudaStreamCreate") ||
        !cuda_ok(c, cudaEventCreateWithFlags(&l.scratch_free, cudaEventDisableTiming), "cudaEventCreate"))
      return fail(RPL_RESULT_OPERATION_FAIL);
    const size_t fast_nodes = (size_t)c->fast_grid * max_nodes;  // launch_scan_fast never gets a larger grid
    const size_t gen_nodes = (size_t)c->general_grid * max_nodes;
    l.fws.max_nodes = max_nodes;
    l.gws.max_nodes = max_nodes;
    if (!cuda_ok(c, dev_alloc(&l.fallback_list, max_scans), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.fallback_count, 4), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.fws.group, fast_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.gws.keyf, gen_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.gws.idx0, gen_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.gws.idx1, gen_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.gws.vidx, gen_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&l.gws.cell, gen_nodes), "cudaMalloc"))
      return fail(oom);
    if (i == 0) {
      if (!cuda_ok(c, rpl::cloud_workspace_alloc(l.cws, c->num_sms, max_nodes), "cloud workspace")) return fail(oom);
      l.owns_cws = true;
    } else {  // read-only tables shared with lane 0; the PointCloud2 post passes run on lane 0 only
      l.cws = rpl::CloudWorkspace{};
      l.cws.trig = c->lane[0].cws.trig;
      l.cws.angle = c->lane[0].cws.angle;
    }
    if (!cuda_ok(c, cudaMemset(l.fallback_count, 0, 4 * sizeof(uint32_t)), "cudaMemset"))
      return fail(RPL_RESULT_OPERATION_FAIL);
  }
  if (!cuda_ok(c, cudaHostAlloc(reinterpret_cast<void**>(&c->h_counts), (size_t)max_scans * 4, cudaHostAllocDefault),
               "cudaHostAlloc") ||
      !cuda_ok(c, cudaHostAlloc(reinterpret_cast<void**>(&c->h_small), (size_t)max_scans * 16, cudaHostAllocDefault),
               "cudaHostAlloc"))
    return fail(RPL_RESULT_INSUFFICIENT_MEMORY);
  {
    c->one_stride = ((size_t)max_nodes + 1) & ~(size_t)1;
    const size_t bytes = c->one_stride * (8 + 8 + 4 + 4) + 64;
    if (!cuda_ok(c, cudaHostAlloc(reinterpret_cast<void**>(&c->h_one), bytes, cudaHostAllocDefault), "cudaHostAlloc") ||
        !cuda_ok(c, cudaMalloc(reinterpret_cast<void**>(&c->d_one), bytes), "cudaMalloc"))
      return fail(RPL_RESULT_INSUFFICIENT_MEMORY);
  }
  *out = c;
  return RPL_RESULT_OK;
}

void rpl_ctx_destroy(rpl_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  for (int i = 0; i < kLanes; ++i) {
    if (c->lane[i].stream) cudaStreamSynchronize(c->lane[i].stream);
    free_lane(c->lane[i]);
  }
  if (c->asm_done) cudaEventDestroy(c->asm_done);
  cudaFree(c->prof_stamps);
  cudaFree(c->d_reset_prefix);
  cudaFree(c->d_desc);
  if (c->h_one) cudaFreeHost(c->h_one);
  cudaFree(c->d_one);
  if (c->h_counts) cudaFreeHost(c->h_counts);
  if (c->h_small) cudaFreeHost(c->h_small);
  delete c;
}

const char* rpl_last_error(const rpl_ctx* c) { return c ? c->err.c_str() : "null context"; }

rpl_result rpl_ctx_synchronize(rpl_ctx* c) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  for (int i = 0; i < kLanes; ++i)
    RPL_CUDA(c, cudaStreamSynchronize(c->lane[i].stream), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_host_alloc(size_t bytes, void** out) {
  if (!out) return RPL_RESULT_INVALID_DATA;
  *out = nullptr;
  return cudaHostAlloc(out, std::max<size_t>(bytes, 1), cudaHostAllocDefault) == cudaSuccess
             ? RPL_RESULT_OK
             : RPL_RESULT_INSUFFICIENT_MEMORY;
}
void rpl_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

uint64_t rpl_ctx_launch_count(const rpl_ctx* c) { return c ? c->launches : 0; }

rpl_result rpl_ctx_profile(rpl_ctx* c, int enable) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (enable && !c->prof_stamps) {
    RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&c->prof_stamps), rpl_ctx::kProfStamps * 16),
             RPL_RESULT_INSUFFICIENT_MEMORY);
    c->prof_stamps_used = rpl_ctx::kProfStamps;  // the drain initialises every record
    const rpl_result r = prof_drain(c);
    if (r != RPL_RESULT_OK) return r;
  }
  c->profile = enable != 0;
  return RPL_RESULT_OK;
}

rpl_result rpl_ctx_profile_read(rpl_ctx* c, double* fast_ms, uint32_t* fast_launches,
                                double* general_ms, uint32_t* general_launches) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  const rpl_result r = prof_drain(c);
  if (r != RPL_RESULT_OK) return r;
  if (fast_ms) *fast_ms = c->prof_ms[0];
  if (fast_launches) *fast_launches = c->prof_n[0];
  if (general_ms) *general_ms = c->prof_ms[1];
  if (general_launches) *general_launches = c->prof_n[1];
  c->prof_ms[0] = c->prof_ms[1] = 0.0;
  c->prof_n[0] = c->prof_n[1] = 0;
  return RPL_RESULT_OK;
}

// ---- device-resident batch ----------------------------------------------------------------
rpl_result rpl_scan_batch_dev(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                              uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                              rpl_node_hq* nodes_out, float* ranges, float* intensities,
                              uint32_t* beam_counts, float* angle_increment, uint32_t* status,
                              uint32_t* path, void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (n_scans != 0 && stride == 0) {
    c->err = "stride == 0";
    return RPL_RESULT_INVALID_DATA;
  }
  // counts[] live on the device: a scan with counts[s] > stride or > the context's max_nodes is reported
  // through status[s] = RPL_RESULT_INVALID_DATA by the kernels (nothing else is written for it)
  return enqueue_scan(c, c->lane[0], nodes, counts, n_scans, stride, params, nodes_out, ranges,
                      intensities, beam_counts, angle_increment, status, path, st);
}

static_assert(sizeof(rpl_scan_filter_settings) == 68 && sizeof(rpl::ScanFilter) == sizeof(rpl_scan_filter_settings) &&
                  offsetof(rpl_scan_filter_settings, range_lo) == offsetof(rpl::ScanFilter, range_lo) &&
                  offsetof(rpl_scan_filter_settings, shadow_angle) == offsetof(rpl::ScanFilter, shadow_tan) &&
                  offsetof(rpl_scan_filter_settings, speckle_window) == offsetof(rpl::ScanFilter, speckle_window) &&
                  offsetof(rpl_scan_filter_settings, enabled) == 64,
              "rpl::ScanFilter must be laid out as rpl_scan_filter_settings, tan(shadow_angle) for shadow_angle");
static_assert(sizeof(rpl_scan_footprint) == 544 && offsetof(rpl_scan_footprint, y) == 256 &&
                  offsetof(rpl_scan_footprint, n_vertices) == 512 && offsetof(rpl_scan_footprint, invert) == 528 &&
                  offsetof(rpl_scan_footprint, pose_x) == 532 && offsetof(rpl_scan_footprint, pose_y) == 536 &&
                  offsetof(rpl_scan_footprint, pose_yaw) == 540,
              "rpl_scan_footprint's layout is the header's");

namespace {

// the limits of rpl_scan_filter_settings (oracle/scan_filter_oracle.py settings_ok)
bool scan_filter_ok(rpl_ctx* c, const rpl_scan_filter_settings& e) {
  bool nan = std::isnan(e.range_lo) || std::isnan(e.range_hi) || std::isnan(e.intensity_min) ||
             std::isnan(e.speckle_max_diff) || std::isnan(e.shadow_angle);
  for (int k = 0; k < 4; ++k) nan = nan || std::isnan(e.mask_lo[k]) || std::isnan(e.mask_hi[k]);
  const char* why = nullptr;
  if (nan) why = "a scan filter parameter is NaN";
  else if (e.speckle_window > rpl::kScanFilterMaxWindow || e.shadow_window > rpl::kScanFilterMaxWindow)
    why = "speckle_window and shadow_window must be <= 16";
  else if (e.speckle_min_neighbours > 2 * e.speckle_window) why = "speckle_min_neighbours > 2 * speckle_window";
  else if (!(e.range_lo <= e.range_hi)) why = "range_lo > range_hi";
  else if (e.shadow_window > 0 && !((double)e.shadow_angle > 0.0 && (double)e.shadow_angle < M_PI / 2))
    why = "shadow_angle must be in (0, pi/2)";
  if (why) c->err = why;
  return why == nullptr;
}

// an entry as the kernel reads it: tan(shadow_angle) in double, rounded to float, once
rpl::ScanFilter scan_filter_entry(const rpl_scan_filter_settings& e) {
  rpl::ScanFilter f{};
  std::memcpy(&f, &e, offsetof(rpl_scan_filter_settings, enabled));
  f.shadow_tan = (float)std::tan((double)e.shadow_angle);
  f.enabled = e.enabled ? 1u : 0u;
  return f;
}

// the limits of rpl_scan_footprint (oracle/scan_footprint_oracle.py footprint_ok)
bool scan_footprint_ok(rpl_ctx* c, const rpl_scan_footprint& e) {
  constexpr float kMax = 1000.0f;
  const char* why = nullptr;
  if (!std::isfinite(e.pose_x) || !std::isfinite(e.pose_y) || !std::isfinite(e.pose_yaw))
    why = "a footprint pose is not finite";
  else if (std::fabs(e.pose_x) > kMax || std::fabs(e.pose_y) > kMax)
    why = "a footprint pose coordinate is beyond 1000 m";
  for (uint32_t p = 0; p < rpl::kFootprintMaxPolygons && !why; ++p) {
    const uint32_t n = e.n_vertices[p];
    if (n != 0 && (n < 3 || n > rpl::kFootprintMaxVertices)) {
      why = "a footprint polygon's n_vertices must be 0 or 3..16";
      break;
    }
    for (uint32_t k = 0; k < n; ++k)
      if (!(std::fabs(e.x[p][k]) <= kMax && std::fabs(e.y[p][k]) <= kMax)) {
        why = "a footprint vertex is not finite or beyond 1000 m";
        break;
      }
  }
  if (why) c->err = why;
  return why == nullptr;
}

// a footprint as the kernel reads it: the used polygons first, each vertex moved into the scan frame in double (every
// operation rounded as written) and rounded to float once
rpl::ScanFootprint scan_footprint_entry(const rpl_scan_footprint& e) {
  rpl::ScanFootprint f{};
  const double c = std::cos((double)e.pose_yaw), s = std::sin((double)e.pose_yaw);
  const double px = e.pose_x, py = e.pose_y;
  for (uint32_t p = 0; p < rpl::kFootprintMaxPolygons; ++p) {
    const uint32_t n = e.n_vertices[p];
    if (n == 0) continue;
    const uint32_t q = f.n_polygons++;
    for (uint32_t k = 0; k < n; ++k) {
      const double dx = (double)e.x[p][k] - px, dy = (double)e.y[p][k] - py;
      f.x[q][k] = (float)(c * dx + s * dy);
      f.y[q][k] = (float)(-s * dx + c * dy);
    }
    f.n_vertices[q] = n;
    f.invert[q] = e.invert[p] ? 1u : 0u;
  }
  return f;
}

}  // namespace

rpl_result rpl_scan_filter_batch_dev(rpl_ctx* c, const rpl_scan_filter_settings* settings, float* ranges,
                                     const float* intensities, const uint32_t* beam_counts,
                                     const float* angle_increment, uint32_t n_scans, uint32_t stride, void* stream) {
  return rpl_scan_filter_footprint_batch_dev(c, settings, nullptr, ranges, intensities, beam_counts, angle_increment,
                                             n_scans, stride, stream);
}

rpl_result rpl_scan_filter_footprint_batch_dev(rpl_ctx* c, const rpl_scan_filter_settings* settings,
                                               const rpl_scan_footprint* footprint, float* ranges,
                                               const float* intensities, const uint32_t* beam_counts,
                                               const float* angle_increment, uint32_t n_scans, uint32_t stride,
                                               void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (!settings || !ranges || !intensities || !beam_counts || !angle_increment) {
    c->err = "null settings, ranges, intensities, beam_counts or angle_increment";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_scans != 0 && (stride == 0 || stride > rpl::kScanFilterMaxBeams)) {
    c->err = "stride must be in [1, 8192]";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!scan_filter_ok(c, *settings)) return RPL_RESULT_INVALID_DATA;
  if (footprint && !scan_footprint_ok(c, *footprint)) return RPL_RESULT_INVALID_DATA;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (!settings->enabled || n_scans == 0) return RPL_RESULT_OK;
  rpl::ScanFilterArgs a{};
  a.one = scan_filter_entry(*settings);
  if (footprint) a.one_footprint = scan_footprint_entry(*footprint);
  a.ranges = ranges;
  a.intensities = intensities;
  a.stride = stride;
  a.beam_counts = beam_counts;
  a.angle_increment = angle_increment;
  a.n_scans = n_scans;
  RPL_CUDA(c, rpl::launch_scan_filter(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

static_assert(sizeof(rpl_scan_cloud_params) == 8 && offsetof(rpl_scan_cloud_params, range_cutoff) == 4 &&
                  RPL_SCAN_CLOUD_INTENSITY == rpl::kScanCloudIntensity && RPL_SCAN_CLOUD_INDEX == rpl::kScanCloudIndex &&
                  RPL_SCAN_CLOUD_DISTANCE == rpl::kScanCloudDistance &&
                  RPL_SCAN_CLOUD_TIMESTAMP == rpl::kScanCloudTimestamp,
              "rpl_scan_cloud_params and its channel bits are the header's");
static_assert(sizeof(rpl_scan_cloud_transform) == 64 && offsetof(rpl_scan_cloud_transform, rotation) == 24 &&
                  offsetof(rpl_scan_cloud_transform, enabled) == 56 &&
                  RPL_SCAN_CLOUD_VIEWPOINT == rpl::kScanCloudViewpoint &&
                  RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS == rpl::kScanCloudPerStreamTransforms,
              "rpl_scan_cloud_transform and the transform bits are the header's");
static_assert(sizeof(rpl_rescan_settings) == 40 && offsetof(rpl_rescan_settings, angle_max) == 4 &&
                  offsetof(rpl_rescan_settings, angle_increment) == 8 && offsetof(rpl_rescan_settings, range_min) == 12 &&
                  offsetof(rpl_rescan_settings, range_max) == 16 && offsetof(rpl_rescan_settings, min_height) == 20 &&
                  offsetof(rpl_rescan_settings, max_height) == 24 && offsetof(rpl_rescan_settings, inf_epsilon) == 28 &&
                  offsetof(rpl_rescan_settings, scan_time) == 32 && offsetof(rpl_rescan_settings, use_inf) == 36 &&
                  offsetof(rpl_rescan_settings, enabled) == 37,
              "rpl_rescan_settings is the header's");
static_assert(sizeof(rpl_rescan_window) == 8 && offsetof(rpl_rescan_window, observations) == 0 &&
                  offsetof(rpl_rescan_window, statistic) == 4 && RPL_RESCAN_WINDOW_MEDIAN == rpl::kRescanWindowMedian &&
                  RPL_RESCAN_WINDOW_MEAN == rpl::kRescanWindowMean,
              "rpl_rescan_window is the header's");
static_assert(sizeof(rpl_msgs_out) == 40 && offsetof(rpl_msgs_out, capacity) == 8 &&
                  offsetof(rpl_msgs_out, msg_offsets) == 16 && offsetof(rpl_msgs_out, msg_sizes) == 24 &&
                  offsetof(rpl_msgs_out, total_bytes) == 32,
              "rpl_msgs_out is the header's");

namespace {

// the rules of rpl_scan_cloud_params (oracle/scan_cloud_oracle.py params_ok); `extra`: the bits beyond the four
// channels the call accepts (the viewpoint and the per-stream transforms, where a transform applies)
bool scan_cloud_ok(rpl_ctx* c, const rpl_scan_cloud_params& p, uint32_t extra = 0) {
  const char* why = nullptr;
  if (p.channels & ~(rpl::kScanCloudChannels | extra))
    why = extra ? "unknown scan cloud channel bits, or RPL_SCAN_CLOUD_VIEWPOINT without a transform"
                : "unknown scan cloud channel bits (only 0x01, 0x02, 0x04, 0x08)";
  else if (std::isnan(p.range_cutoff)) why = "range_cutoff is NaN";
  if (why) c->err = why;
  return why == nullptr;
}

uint32_t scan_cloud_point_step(uint32_t channels) {
  return 12u + 4u * (uint32_t)__builtin_popcount(channels & rpl::kScanCloudChannels) +
         ((channels & rpl::kScanCloudViewpoint) ? 12u : 0u);
}

// The PointCloud2 members between the header and the data of fields names[0..nf) (datatypes types[], count 1, offsets
// 4 bytes apart from 0): height 1, width, the fields, is_bigendian 0, point_step, row_step, data length
extern "C++" template <class Tail>
Tail pointcloud2_tail(const char* const* names, const uint8_t* types, uint32_t nf, uint32_t point_step) {
  Tail t{};
  uint8_t* b = reinterpret_cast<uint8_t*>(t.w);
  uint32_t n = 0;
  auto u32 = [&](uint32_t v) {
    n = (n + 3) & ~3u;
    std::memcpy(b + n, &v, 4);
    n += 4;
  };
  u32(1);
  t.at_width = n / 4;
  u32(0);
  u32(nf);
  for (uint32_t f = 0; f < nf; ++f) {
    const uint32_t L = (uint32_t)std::strlen(names[f]);
    u32(L + 1);
    std::memcpy(b + n, names[f], L + 1);
    n += L + 1;
    u32(4 * f);
    b[n++] = types[f];
    u32(1);
  }
  b[n++] = 0;  // is_bigendian
  u32(point_step);
  t.at_row_step = (n + 3) / 4;
  u32(0);
  t.at_data = n / 4;
  u32(0);
  t.bytes = n;
  return t;
}

// the tails of the channel sets below `sets`: x, y, z, then laser_geometry's channels in bit order, then the viewpoint's
// three fields
extern "C++" template <class Tail>
std::vector<Tail> scan_cloud_tails(uint32_t sets) {
  std::vector<Tail> v(sets);
  const char* const channel_names[7] = {"intensity", "index", "distances", "stamps", "vp_x", "vp_y", "vp_z"};
  const uint8_t channel_types[7] = {7, 5, 7, 7, 7, 7, 7};  // FLOAT32, INT32, FLOAT32 ...
  for (uint32_t ch = 0; ch < sets; ++ch) {
    const char* names[10] = {"x", "y", "z"};
    uint8_t types[10] = {7, 7, 7};
    uint32_t nf = 3;
    for (uint32_t k = 0; k < 7; ++k)
      if (ch & (1u << (k < 4 ? k : 4))) {
        names[nf] = channel_names[k];
        types[nf++] = channel_types[k];
      }
    v[ch] = pointcloud2_tail<Tail>(names, types, nf, scan_cloud_point_step(ch));
  }
  return v;
}
const rpl::ScanCloudTail& scan_cloud_tail(uint32_t channels) {
  static const std::vector<rpl::ScanCloudTail> tails = scan_cloud_tails<rpl::ScanCloudTail>(rpl::kScanCloudChannels + 1);
  return tails[channels];
}
// a transforming call's: every channel set with or without the viewpoint
const rpl::ScanCloudTailXf& scan_cloud_tail_xf(uint32_t channels) {
  static const std::vector<rpl::ScanCloudTailXf> tails =
      scan_cloud_tails<rpl::ScanCloudTailXf>(2 * rpl::kScanCloudViewpoint);
  return tails[channels & (rpl::kScanCloudChannels | rpl::kScanCloudViewpoint)];
}
// its tail's bytes
uint32_t scan_cloud_tail_bytes(uint32_t channels) {
  return (channels & rpl::kScanCloudPerStreamTransforms) ? scan_cloud_tail_xf(channels).bytes
                                                         : scan_cloud_tail(channels).bytes;
}

// the settings of params into a (a call with RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS: the transforming kernel's tail; the
// caller gives it the tables)
void scan_cloud_setup(rpl::ScanCloudArgs& a, const rpl_scan_cloud_params& p) {
  a.channels = p.channels;
  a.point_step = scan_cloud_point_step(p.channels);
  a.range_cutoff = p.range_cutoff;
  if (p.channels & rpl::kScanCloudPerStreamTransforms) {
    a.transform = 1;
    a.tail_xf = scan_cloud_tail_xf(p.channels);
  } else {
    a.tail = scan_cloud_tail(p.channels);
  }
}

// The limits of one transform entry (tests/scan_cloud_transform_oracle.py transform_ok); frame: its target frame, or
// nullptr where none is given (the stateless call)
bool scan_cloud_transform_ok(rpl_ctx* c, const rpl_scan_cloud_transform& e, const char* frame, bool framed) {
  const char* why = nullptr;
  const double* q = e.rotation;
  bool finite = true;
  for (int k = 0; k < 3; ++k) finite = finite && std::isfinite(e.translation[k]);
  for (int k = 0; k < 4; ++k) finite = finite && std::isfinite(q[k]);
  if (!finite) why = "a transform's translation and rotation must be finite";
  else if (!(std::fabs(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] - 1.0) <= 1e-3))
    why = "a transform's quaternion must be of norm 1 (|x^2 + y^2 + z^2 + w^2 - 1| <= 1e-3)";
  else if (!(std::fabs(e.translation[0]) <= 1000.0 && std::fabs(e.translation[1]) <= 1000.0 &&
             std::fabs(e.translation[2]) <= 1000.0))
    why = "a transform's translation must be within 1000 m";
  else if (framed && !frame) why = "null target_frames[s] of an enabled entry";
  if (why) {
    c->err = why;
    return false;
  }
  return !framed || frame_id_length_ok(c, std::strlen(frame));
}

// The rows {R_k0, R_k1, t_k, on} of a transform entry (scan_cloud_kernel<true>): R from the quaternion in double as
// tf2's Matrix3x3::setRotation, each entry and t rounded to float once; a disabled entry's are zero (on 0: no
// transform)
void scan_cloud_rows(const rpl_scan_cloud_transform& e, float4 rows[3]) {
  if (!e.enabled) {
    for (int k = 0; k < 3; ++k) rows[k] = float4{0.0f, 0.0f, 0.0f, 0.0f};
    return;
  }
  const double x = e.rotation[0], y = e.rotation[1], z = e.rotation[2], w = e.rotation[3];
  const double d = x * x + y * y + z * z + w * w, s = 2.0 / d;
  const double xs = x * s, ys = y * s, zs = z * s;
  const double wx = w * xs, wy = w * ys, wz = w * zs;
  const double xx = x * xs, xy = x * ys, xz = x * zs;
  const double yy = y * ys, yz = y * zs, zz = z * zs;
  const double R[3][2] = {{1.0 - (yy + zz), xy - wz}, {xy + wz, 1.0 - (xx + zz)}, {xz - wy, yz + wx}};
  for (int k = 0; k < 3; ++k)
    rows[k] = float4{(float)R[k][0], (float)R[k][1], (float)e.translation[k], 1.0f};
}

}  // namespace

rpl_result rpl_scan_cloud_transform_batch_dev(rpl_ctx* c, const rpl_scan_cloud_params* params,
                                              const rpl_scan_cloud_transform* transform, const float* ranges,
                                              const float* intensities, const uint32_t* beam_counts,
                                              const float* angle_increment, const float* time_increment,
                                              float range_min, float range_max, uint32_t n_scans, uint32_t stride,
                                              void* points, uint32_t* point_counts, void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (!params || !ranges || !intensities || !beam_counts || !angle_increment || !points || !point_counts) {
    c->err = "null params, ranges, intensities, beam_counts, angle_increment, points or point_counts";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!scan_cloud_ok(c, *params, transform ? rpl::kScanCloudViewpoint : 0u)) return RPL_RESULT_INVALID_DATA;
  if (transform && transform->enabled && !scan_cloud_transform_ok(c, *transform, nullptr, false))
    return RPL_RESULT_INVALID_DATA;
  if (n_scans != 0 && (stride == 0 || stride > c->max_nodes)) {
    c->err = "stride must be in [1, the context's max_nodes]";
    return RPL_RESULT_INVALID_DATA;
  }
  if (reinterpret_cast<uintptr_t>(points) & 3u) {
    c->err = "points must be 4-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (n_scans == 0) return RPL_RESULT_OK;
  rpl::ScanCloudArgs a{};
  scan_cloud_setup(a, *params);
  a.m.counts = beam_counts;
  a.m.ranges = ranges;
  a.m.intensities = intensities;
  a.m.angle_increment = angle_increment;
  a.m.stride = stride;
  a.m.n = n_scans;
  a.range_min = range_min;
  a.range_max = range_max;
  a.time_increment = time_increment;
  a.kept = point_counts;
  a.points = static_cast<float*>(points);
  if (transform) {
    a.transform = 1;
    scan_cloud_rows(*transform, a.xf_one);
  }
  RPL_CUDA(c, rpl::launch_scan_cloud(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

rpl_result rpl_scan_cloud_batch_dev(rpl_ctx* c, const rpl_scan_cloud_params* params, const float* ranges,
                                    const float* intensities, const uint32_t* beam_counts,
                                    const float* angle_increment, const float* time_increment, float range_min,
                                    float range_max, uint32_t n_scans, uint32_t stride, void* points,
                                    uint32_t* point_counts, void* stream) {
  return rpl_scan_cloud_transform_batch_dev(c, params, nullptr, ranges, intensities, beam_counts, angle_increment,
                                            time_increment, range_min, range_max, n_scans, stride, points,
                                            point_counts, stream);
}

namespace {

// ranges_size of an entry: ceil(fl32(fl32(angle_max - angle_min) / angle_increment)), the package's float arithmetic
// (oracle/rescan_oracle.py ranges_size); 0 when it is not a count
uint32_t rescan_bins(const rpl_rescan_settings& e) {
  const float q = std::ceil((e.angle_max - e.angle_min) / e.angle_increment);
  return q >= 1.0f && q <= (float)rpl::kRescanMaxBins ? (uint32_t)q : 0u;
}

// the limits of an entry (oracle/rescan_oracle.py settings_ok)
bool rescan_ok(rpl_ctx* c, const rpl_rescan_settings& e) {
  const float v[9] = {e.angle_min, e.angle_max, e.angle_increment, e.range_min, e.range_max,
                      e.min_height, e.max_height, e.inf_epsilon, e.scan_time};
  const char* why = nullptr;
  if (!std::all_of(v, v + 9, [](float f) { return std::isfinite(f); })) why = "a rescan entry's floats must be finite";
  else if (!(e.angle_increment > 0.0f) || !(e.angle_min < e.angle_max))
    why = "a rescan entry needs angle_increment > 0 and angle_min < angle_max";
  else if (rescan_bins(e) == 0) why = "a rescan entry's ranges_size must be in [1, 8192]";
  else if (!(0.0f <= e.range_min && e.range_min <= e.range_max)) why = "a rescan entry needs 0 <= range_min <= range_max";
  else if (!(e.min_height <= e.max_height)) why = "a rescan entry needs min_height <= max_height";
  else if (!(e.inf_epsilon >= 0.0f)) why = "a rescan entry needs inf_epsilon >= 0";
  if (why) c->err = why;
  return why == nullptr;
}

// an entry as rescan_kernel reads it (a disabled one: no bins, no message)
rpl::RescanGrid rescan_grid(const rpl_rescan_settings& e, bool use_enabled) {
  rpl::RescanGrid g{};
  if (use_enabled && !e.enabled) return g;
  g.angle_min = e.angle_min;
  g.angle_max = e.angle_max;
  g.angle_increment = e.angle_increment;
  g.range_min = e.range_min;
  g.range_max = e.range_max;
  g.min_height = e.min_height;
  g.max_height = e.max_height;
  g.scan_time = e.scan_time;
  const float seed = e.use_inf ? INFINITY : (float)((double)e.range_max + (double)e.inf_epsilon);
  std::memcpy(&g.seed, &seed, 4);
  g.bins = rescan_bins(e);
  return g;
}

}  // namespace

rpl_result rpl_rescan_batch_dev(rpl_ctx* c, const rpl_rescan_settings* settings,
                                const rpl_scan_cloud_params* cloud_params, const rpl_scan_cloud_transform* transform,
                                const float* ranges, const float* intensities, const uint32_t* beam_counts,
                                const float* angle_increment, float range_min, float range_max, uint32_t n_scans,
                                uint32_t stride, float* out_ranges, void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (!settings || !cloud_params || !ranges || !beam_counts || !angle_increment || !out_ranges) {
    c->err = "null settings, cloud_params, ranges, beam_counts, angle_increment or out_ranges";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!rescan_ok(c, *settings)) return RPL_RESULT_INVALID_DATA;
  if (!scan_cloud_ok(c, *cloud_params, transform ? rpl::kScanCloudViewpoint : 0u)) return RPL_RESULT_INVALID_DATA;
  if (transform && transform->enabled && !scan_cloud_transform_ok(c, *transform, nullptr, false))
    return RPL_RESULT_INVALID_DATA;
  if (n_scans != 0 && (stride == 0 || stride > c->max_nodes)) {
    c->err = "stride must be in [1, the context's max_nodes]";
    return RPL_RESULT_INVALID_DATA;
  }
  if (reinterpret_cast<uintptr_t>(out_ranges) & 3u) {
    c->err = "out_ranges must be 4-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (n_scans == 0) return RPL_RESULT_OK;
  rpl::RescanArgs a{};
  a.c.channels = cloud_params->channels;
  a.c.range_cutoff = cloud_params->range_cutoff;
  a.c.m.counts = beam_counts;
  a.c.m.ranges = ranges;
  a.c.m.angle_increment = angle_increment;
  a.c.m.stride = stride;
  a.c.m.n = n_scans;
  a.c.range_min = range_min;
  a.c.range_max = range_max;
  if (transform) {
    a.c.transform = 1;
    scan_cloud_rows(*transform, a.c.xf_one);
  }
  a.grid_one = rescan_grid(*settings, false);
  a.out = out_ranges;
  RPL_CUDA(c, rpl::launch_rescan(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

namespace {

// the limits of a window (oracle/rescan_window_oracle.py window_ok)
bool rescan_window_ok(rpl_ctx* c, const rpl_rescan_window& w) {
  if (w.observations >= 1 && w.observations <= rpl::kRescanWindowMax &&
      (w.statistic == RPL_RESCAN_WINDOW_MEDIAN || w.statistic == RPL_RESCAN_WINDOW_MEAN))
    return true;
  c->err = "a rescan window needs observations in [1, 16] and statistic RPL_RESCAN_WINDOW_MEDIAN or _MEAN";
  return false;
}

}  // namespace

rpl_result rpl_rescan_window_batch_dev(rpl_ctx* c, const rpl_rescan_window* window, const float* in, uint32_t n_scans,
                                       uint32_t bins, float* out, void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (!window || !in || !out) {
    c->err = "null window, in or out";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!rescan_window_ok(c, *window)) return RPL_RESULT_INVALID_DATA;
  if (bins == 0 || bins > rpl::kRescanMaxBins) {
    c->err = "bins must be in [1, 8192]";
    return RPL_RESULT_INVALID_DATA;
  }
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 3u) {
    c->err = "in and out must be 4-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (n_scans == 0) return RPL_RESULT_OK;
  RPL_CUDA(c, rpl::launch_rescan_window_batch(in, n_scans, bins, window->observations, window->statistic, out,
                                              c->num_sms, st),
           RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

rpl_result rpl_rescan_merge_batch_dev(rpl_ctx* c, const rpl_rescan_settings* settings, const float* in,
                                      const uint32_t* row_group, uint32_t n_rows, uint32_t n_groups, float* out,
                                      void* stream) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (!settings || !out || (n_rows && (!in || !row_group))) {
    c->err = "null settings, in, row_group or out";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!rescan_ok(c, *settings)) return RPL_RESULT_INVALID_DATA;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(row_group) | reinterpret_cast<uintptr_t>(out)) & 3u) {
    c->err = "in, row_group and out must be 4-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  const rpl::RescanGrid g = rescan_grid(*settings, false);
  if ((unsigned long long)n_groups * g.bins == 0) return RPL_RESULT_OK;
  RPL_CUDA(c, rpl::launch_rescan_merge_batch(in, row_group, n_rows, n_groups, g.bins, g.seed, out, c->num_sms, st),
           RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// ---- host-buffer batch: chunked over the two lanes so that the H2D copy of chunk i+1, the
// kernels of chunk i and the D2H copy of chunk i-1 overlap ---------------------------------
rpl_result rpl_scan_batch(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                          uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                          rpl_node_hq* nodes_out, float* ranges, float* intensities,
                          uint32_t* beam_counts, float* angle_increment, uint32_t* status,
                          uint32_t* path) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (n_scans == 0) return RPL_RESULT_OK;
  if (!nodes || !counts || !params) {
    c->err = "null nodes/counts/params";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_scans > c->max_scans || stride == 0) {
    c->err = "n_scans exceeds max_scans (or stride == 0)";
    return RPL_RESULT_INVALID_DATA;
  }
  for (uint32_t s = 0; s < n_scans; ++s)
    if (counts[s] > stride || counts[s] > c->max_nodes) {
      c->err = "counts[s] exceeds stride or the context's max_nodes";
      return RPL_RESULT_INVALID_DATA;
    }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);

  // chunk: about 32 MiB of nodes, at least one scan
  const size_t target_nodes = (32u << 20) / sizeof(rpl_node_hq);
  uint32_t chunk = (uint32_t)std::max<size_t>(1, target_nodes / stride);
  chunk = std::min(chunk, n_scans);
  const bool want_scan = ranges != nullptr;
  struct Regions {
    rpl_node_hq *nodes, *nodes_out;
    float *ranges, *intens, *inc;
    uint32_t *counts, *beams, *status, *path;
  };
  auto layout = [&, cnt = (size_t)chunk * stride](Carve& k) {
    const size_t scan = want_scan ? cnt : 0;
    return Regions{k.take<rpl_node_hq>(cnt), k.take<rpl_node_hq>(nodes_out ? cnt : 0), k.take<float>(scan),
                   k.take<float>(scan), k.take<float>(chunk), k.take<uint32_t>(chunk), k.take<uint32_t>(chunk),
                   k.take<uint32_t>(chunk), k.take<uint32_t>(chunk)};
  };
  if (const rpl_result r = grow_stage(c, kLanes, layout); r != RPL_RESULT_OK) return r;
  const cudaMemcpyKind h2d = cudaMemcpyHostToDevice, d2h = cudaMemcpyDeviceToHost;
  std::memcpy(c->h_counts, counts, (size_t)n_scans * sizeof(uint32_t));
  uint32_t* hs_beams = c->h_small;
  uint32_t* hs_inc = c->h_small + c->max_scans;
  uint32_t* hs_status = c->h_small + 2 * (size_t)c->max_scans;
  uint32_t* hs_path = c->h_small + 3 * (size_t)c->max_scans;
  // one chunk through one lane
  auto run_chunk = [&](Lane& l, uint32_t s0, uint32_t ns) -> rpl_result {
    const size_t off = (size_t)s0 * stride, cnt = (size_t)ns * stride;
    Carve k{l.stage};
    const Regions d = layout(k);
    // the lane's previous chunk (2 chunks ago) must have left its staging buffers
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(d.nodes, nodes + off, cnt * sizeof(rpl_node_hq), h2d, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(d.counts, c->h_counts + s0, ns * sizeof(uint32_t), h2d, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    // The kernels write only the first counts[s] nodes of a scan they ascend (nothing for an empty or
    // unmeasured scan: the reference leaves those buffers untouched).  The whole [ns][stride] region goes
    // back to the caller, so it starts out as the caller's own bytes, not as leftovers of an earlier chunk.
    if (nodes_out && params->apply_ascend)
      RPL_CUDA(c, cudaMemcpyAsync(d.nodes_out, d.nodes, cnt * sizeof(rpl_node_hq), cudaMemcpyDeviceToDevice, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    rpl_result r = enqueue_scan(c, l, d.nodes, d.counts, ns, stride, params, nodes_out ? d.nodes_out : nullptr,
                                want_scan ? d.ranges : nullptr, want_scan ? d.intens : nullptr, d.beams, d.inc,
                                d.status, d.path, l.stream);
    if (r != RPL_RESULT_OK) return r;
    if (nodes_out)
      RPL_CUDA(c, cudaMemcpyAsync(nodes_out + off, d.nodes_out, cnt * sizeof(rpl_node_hq), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    if (want_scan) {
      RPL_CUDA(c, cudaMemcpyAsync(ranges + off, d.ranges, cnt * sizeof(float), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(intensities + off, d.intens, cnt * sizeof(float), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    }
    if (beam_counts)
      RPL_CUDA(c, cudaMemcpyAsync(hs_beams + s0, d.beams, ns * sizeof(uint32_t), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    if (angle_increment)
      RPL_CUDA(c, cudaMemcpyAsync(hs_inc + s0, d.inc, ns * sizeof(float), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    if (status)
      RPL_CUDA(c, cudaMemcpyAsync(hs_status + s0, d.status, ns * sizeof(uint32_t), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    if (path)
      RPL_CUDA(c, cudaMemcpyAsync(hs_path + s0, d.path, ns * sizeof(uint32_t), d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    return RPL_RESULT_OK;
  };
  const rpl_result r = run_chunks(c, n_scans, chunk, run_chunk);
  if (r != RPL_RESULT_OK) return r;
  if (beam_counts) std::memcpy(beam_counts, hs_beams, (size_t)n_scans * 4);
  if (angle_increment) std::memcpy(angle_increment, hs_inc, (size_t)n_scans * 4);
  if (status) std::memcpy(status, hs_status, (size_t)n_scans * 4);
  if (path) std::memcpy(path, hs_path, (size_t)n_scans * 4);
  return RPL_RESULT_OK;
}

rpl_result rpl_ascend_scan_batch(rpl_ctx* c, rpl_node_hq* nodes, const uint32_t* counts,
                                 uint32_t n_scans, uint32_t stride, uint32_t* status) {
  rpl_scan_params p{};
  p.apply_ascend = 1;
  return rpl_scan_batch(c, nodes, counts, n_scans, stride, &p, nodes, nullptr, nullptr, nullptr,
                        nullptr, status, nullptr);
}

rpl_result rpl_laserscan_batch(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                               uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                               float* ranges, float* intensities, uint32_t* beam_counts,
                               float* angle_increment) {
  if (!params) return RPL_RESULT_INVALID_DATA;
  rpl_scan_params p = *params;
  p.apply_ascend = 0;  // the LaserScan never depends on the ascended buffer (see DESIGN.md)
  return rpl_scan_batch(c, nodes, counts, n_scans, stride, &p, nullptr, ranges, intensities,
                        beam_counts, angle_increment, nullptr, nullptr);
}

// ---- single scan (the reference-shaped calls) ----------------------------------------------
namespace {

struct OneSmall {  // the 64-byte control block between the input and the outputs
  uint32_t count;
  uint32_t fallback_count;
  uint32_t fallback_list;
  uint32_t beams;
  float inc;
  uint32_t status;
  uint32_t path;
  uint32_t pad[9];
};
static_assert(sizeof(OneSmall) == 64, "control block");

// One lidar revolution: the operating point of the reference (one scan thread, ~10 Hz).  What
// matters here is latency, so the scan travels in one pinned block each way and the general
// kernel is launched only when the fast kernel reports a duplicate-key scan.  The fast kernel is
// the one a batch of one scan at stride one_stride gets (pick_fast).
rpl_result scan_single(rpl_ctx* c, const rpl_node_hq* nodes_in, size_t count, const rpl_scan_params* p,
                       rpl_node_hq* nodes_out, float* ranges, float* intensities, uint32_t* beam_count,
                       float* angle_increment, rpl_result* ascend_status) {
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  Lane& l = c->lane[0];
  const size_t S = c->one_stride, n = count;
  const size_t off_small = S * 8, off_nout = off_small + 64, off_r = off_nout + S * 8, off_i = off_r + S * 4;
  std::memcpy(c->h_one, nodes_in, n * 8);
  OneSmall* hs = reinterpret_cast<OneSmall*>(c->h_one + off_small);
  std::memset(hs, 0, sizeof(OneSmall));
  hs->count = (uint32_t)n;
  // H2D: live nodes + control block (two copies only when the scan is much shorter than max_nodes)
  if (n * 8 + 4096 >= off_small) {
    RPL_CUDA(c, cudaMemcpyAsync(c->d_one, c->h_one, off_small + 64, cudaMemcpyHostToDevice, l.stream),
             RPL_RESULT_OPERATION_FAIL);
  } else {
    RPL_CUDA(c, cudaMemcpyAsync(c->d_one, c->h_one, n * 8, cudaMemcpyHostToDevice, l.stream), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(c->d_one + off_small, hs, 64, cudaMemcpyHostToDevice, l.stream),
             RPL_RESULT_OPERATION_FAIL);
  }
  OneSmall* ds = reinterpret_cast<OneSmall*>(c->d_one + off_small);
  const bool want_nodes = nodes_out != nullptr && p->apply_ascend;
  const bool want_scan = ranges != nullptr;
  rpl::ScanBatchArgs a = scan_args(p, l);
  a.nodes = reinterpret_cast<const uint2*>(c->d_one);  // d_one and S keep bases 16-byte aligned
  a.nodes_out = want_nodes ? reinterpret_cast<uint2*>(c->d_one + off_nout) : nullptr;
  a.counts = &ds->count;
  a.n_scans = 1;
  a.stride = (uint32_t)S;
  a.ranges = want_scan ? reinterpret_cast<float*>(c->d_one + off_r) : nullptr;
  a.intensities = want_scan ? reinterpret_cast<float*>(c->d_one + off_i) : nullptr;
  a.beam_counts = &ds->beams;
  a.angle_inc = &ds->inc;
  a.status = &ds->status;
  a.path = &ds->path;
  a.fallback_list = &ds->fallback_list;  // zeroed by the H2D copy
  a.fallback_count = &ds->fallback_count;
  // D2H extent: control block + whatever was produced, trimmed to the live part
  auto copy_back = [&]() -> rpl_result {
    size_t end = off_nout;
    if (want_nodes) end = off_nout + n * 8;
    if (want_scan) end = off_i + n * 4;
    if (want_scan && (end - off_small) > 3 * (64 + n * 16) + 8192) {
      // short scan in a large context: three small copies beat one copy across the gaps
      RPL_CUDA(c, cudaMemcpyAsync(hs, ds, 64 + (want_nodes ? n * 8 : 0), cudaMemcpyDeviceToHost, l.stream),
               RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(c->h_one + off_r, c->d_one + off_r, n * 4, cudaMemcpyDeviceToHost, l.stream),
               RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(c->h_one + off_i, c->d_one + off_i, n * 4, cudaMemcpyDeviceToHost, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    } else {
      RPL_CUDA(c, cudaMemcpyAsync(hs, ds, end - off_small, cudaMemcpyDeviceToHost, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    }
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);
    return RPL_RESULT_OK;
  };
  // the fallback list is the control block's; fws and gws are lane 0's, which device calls on other streams share
  const FastKernel k = pick_fast(a, p->flags);
  if (k != FastKernel::kNone) {
    rpl_result r = scratch_enter(c, l, l.stream);
    if (r == RPL_RESULT_OK) r = launch_fast(c, l, a, k, l.stream);
    if (r == RPL_RESULT_OK) r = scratch_leave(c, l, l.stream);
    if (r == RPL_RESULT_OK) r = copy_back();
    if (r != RPL_RESULT_OK) return r;
  }
  if (k == FastKernel::kNone || hs->fallback_count != 0) {
    rpl_result r = scratch_enter(c, l, l.stream);
    if (r == RPL_RESULT_OK) r = launch_general(c, l, a, true, l.stream);
    if (r == RPL_RESULT_OK) r = scratch_leave(c, l, l.stream);
    if (r == RPL_RESULT_OK) r = copy_back();
    if (r != RPL_RESULT_OK) return r;
  }
  const uint32_t m = hs->beams;
  if (beam_count) *beam_count = m;
  if (angle_increment) *angle_increment = hs->inc;
  if (ascend_status) *ascend_status = hs->status;
  if (hs->status == RPL_RESULT_INVALID_DATA) return RPL_RESULT_INVALID_DATA;
  if (want_nodes) std::memcpy(nodes_out, c->h_one + off_nout, n * 8);
  if (want_scan && m) {
    std::memcpy(ranges, c->h_one + off_r, (size_t)m * 4);
    std::memcpy(intensities, c->h_one + off_i, (size_t)m * 4);
  }
  return RPL_RESULT_OK;
}

}  // namespace

rpl_result rpl_ascend_scan(rpl_ctx* c, rpl_node_hq* nodes, size_t count) {
  if (!c) return RPL_RESULT_INVALID_DATA;
  if (count == 0) return RPL_RESULT_OPERATION_FAIL;  // reference: i == count -> FAIL
  if (!nodes || count > c->max_nodes) return RPL_RESULT_INVALID_DATA;
  rpl_scan_params p{};
  p.apply_ascend = 1;
  rpl_result status = RPL_RESULT_OPERATION_FAIL;
  rpl_result r = scan_single(c, nodes, count, &p, nodes, nullptr, nullptr, nullptr, nullptr, &status);
  return r != RPL_RESULT_OK ? r : status;
}

rpl_result rpl_laserscan(rpl_ctx* c, const rpl_node_hq* nodes, size_t count,
                         const rpl_scan_params* params, float* ranges, float* intensities,
                         uint32_t* beam_count, float* angle_increment) {
  if (!c || !beam_count || !params) return RPL_RESULT_INVALID_DATA;
  *beam_count = 0;
  if (angle_increment) *angle_increment = 0.0f;
  if (count == 0) return RPL_RESULT_OK;  // publish_scan: nodes.empty() -> return
  if (!nodes || !ranges || !intensities || count > c->max_nodes) return RPL_RESULT_INVALID_DATA;
  rpl_scan_params p = *params;
  p.apply_ascend = 0;  // the LaserScan never depends on the ascended buffer (see DESIGN.md)
  return scan_single(c, nodes, count, &p, nullptr, ranges, intensities, beam_count, angle_increment, nullptr);
}

rpl_result rpl_scan(rpl_ctx* c, rpl_node_hq* nodes, size_t count, const rpl_scan_params* params,
                    float* ranges, float* intensities, uint32_t* beam_count,
                    float* angle_increment, rpl_result* ascend_status) {
  if (!c || !beam_count || !params) return RPL_RESULT_INVALID_DATA;
  *beam_count = 0;
  if (angle_increment) *angle_increment = 0.0f;
  if (ascend_status) *ascend_status = params->apply_ascend ? RPL_RESULT_OPERATION_FAIL : RPL_RESULT_OK;
  if (count == 0) return RPL_RESULT_OK;
  if (!nodes || !ranges || !intensities || count > c->max_nodes) return RPL_RESULT_INVALID_DATA;
  return scan_single(c, nodes, count, params, params->apply_ascend ? nodes : nullptr, ranges, intensities,
                     beam_count, angle_increment, ascend_status);
}

// ---- dense-capsule decode (SURVEY.md 8(f) rank 1) ---------------------------------------------
namespace {
// one launch of the capsule decoder on arguments the entry point has checked (n_streams > 0)
// (list: a mixed byte session's streams of this type, a.n_streams of them)
rpl_result decode_capsules_launch(rpl_ctx* c, uint32_t ans_type, const rpl::CapsuleDecodeArgs& a, void* stream,
                                  const rpl::StreamList* list = nullptr) {
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  // one CTA per stream, up to four (dense) or eight (the other formats) CTAs per SM; a CTA loops over the rest
  const uint32_t ctas_per_sm = ans_type == 0x85 ? 4u : 8u;
  const int grid = (int)std::min<uint32_t>(a.n_streams, (uint32_t)c->num_sms * ctas_per_sm);
  RPL_CUDA(c, rpl::launch_decode_capsules(ans_type, a, grid, st, list), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// one launch of the standard-node decoder on arguments the entry point has checked (n_streams > 0)
rpl_result decode_normal_launch(rpl_ctx* c, const rpl::NormalDecodeArgs& a, void* stream,
                                const rpl::StreamList* list = nullptr) {
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  const int grid = (int)std::min<uint32_t>(a.n_streams, (uint32_t)c->num_sms * 8u);
  RPL_CUDA(c, rpl::launch_decode_normal(a, grid, st, list), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}
}  // namespace

rpl_result rpl_decode_dense_batch_dev(rpl_ctx* c, const uint8_t* capsules, const uint32_t* capsule_counts,
                                      uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                      const uint32_t* sync_state_in, rpl_node_hq* nodes_out,
                                      uint32_t* node_counts, uint32_t* capsule_status,
                                      uint32_t* capsule_node_offset, uint32_t* sync_state_out, void* stream) {
  return rpl_decode_dense_batch_starts_dev(c, capsules, capsule_counts, n_streams, stride_capsules, sample_duration_us,
                                           sync_state_in, nodes_out, node_counts, capsule_status, capsule_node_offset,
                                           sync_state_out, nullptr, 0, nullptr, stream);
}

rpl_result rpl_decode_dense_batch_starts_dev(rpl_ctx* c, const uint8_t* capsules, const uint32_t* capsule_counts,
                                             uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                             const uint32_t* sync_state_in, rpl_node_hq* nodes_out,
                                             uint32_t* node_counts, uint32_t* capsule_status,
                                             uint32_t* capsule_node_offset, uint32_t* sync_state_out,
                                             uint32_t* scan_starts, uint32_t starts_stride, uint32_t* scan_start_counts,
                                             void* stream) {
  if (!c || !capsules || !capsule_counts || !nodes_out) return RPL_RESULT_INVALID_DATA;
  if ((scan_starts == nullptr) != (scan_start_counts == nullptr) || (scan_starts && starts_stride == 0)) {
    c->err = "scan_starts and scan_start_counts go together (starts_stride > 0)";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!sample_duration_ok(c, sample_duration_us)) return RPL_RESULT_INVALID_DATA;
  if ((reinterpret_cast<uintptr_t>(capsules) & 3u) != 0 || misaligned8(nodes_out)) {
    c->err = "capsule buffer must be 4-byte aligned, nodes_out 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_streams == 0) return RPL_RESULT_OK;
  rpl::CapsuleDecodeArgs a{};
  a.capsules = capsules;
  a.counts = capsule_counts;
  a.n_streams = n_streams;
  a.stride_capsules = stride_capsules;
  a.sample_duration_us = sample_duration_us;
  a.state_words = 1;
  a.state_in = sync_state_in;
  a.nodes_out = reinterpret_cast<uint2*>(nodes_out);
  a.node_counts = node_counts;
  a.capsule_status = capsule_status;
  a.capsule_node_offset = capsule_node_offset;
  a.state_out = sync_state_out;
  a.scan_starts = scan_starts;
  a.scan_start_counts = scan_start_counts;
  a.starts_stride = starts_stride;
  return decode_capsules_launch(c, 0x85, a, stream);
}

rpl_result rpl_decode_dense(rpl_ctx* c, const uint8_t* capsules, uint32_t n_capsules, uint32_t sample_duration_us,
                            uint32_t* sync_state, rpl_node_hq* nodes_out, uint32_t* node_count,
                            uint32_t* capsule_status, uint32_t* capsule_node_offset) {
  uint32_t state[2] = {sync_state ? *sync_state : 0u, 0u};
  const rpl_result r = rpl_decode_capsules(c, 0x85, capsules, n_capsules, sample_duration_us, state, nodes_out,
                                           node_count, capsule_status, capsule_node_offset, nullptr, nullptr, nullptr);
  if (r == RPL_RESULT_OK && sync_state) *sync_state = state[0];
  return r;
}

// ---- the other answer formats (SURVEY.md 8(f) rank 1) ----------------------------------------------
uint32_t rpl_capsule_bytes(uint32_t ans_type) {
  switch (ans_type) {
    case 0x82: return 84;
    case 0x83: return 781;
    case 0x84: return 132;
    case 0x85: return 84;
    case 0x86: return 170;
    default: return 0;
  }
}
uint32_t rpl_capsule_nodes(uint32_t ans_type) {
  switch (ans_type) {
    case 0x82: return 32;
    case 0x83: return 96;
    case 0x84: return 96;
    case 0x85: return 40;
    case 0x86: return 64;
    default: return 0;
  }
}

rpl_result rpl_decode_capsules_batch_dev(rpl_ctx* c, uint32_t ans_type, const uint8_t* capsules,
                                         const uint32_t* capsule_counts, uint32_t n_streams,
                                         uint32_t stride_capsules, uint32_t sample_duration_us,
                                         const uint32_t* state_in, rpl_node_hq* nodes_out, uint32_t* node_counts,
                                         uint32_t* capsule_status, uint32_t* capsule_node_offset,
                                         uint32_t* state_out, void* stream) {
  if (!c || !capsules || !capsule_counts || !nodes_out) return RPL_RESULT_INVALID_DATA;
  if (capsule_bytes(c, ans_type) == 0) return RPL_RESULT_INVALID_DATA;
  if (misaligned8(nodes_out)) {
    c->err = "nodes_out must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!sample_duration_ok(c, sample_duration_us)) return RPL_RESULT_INVALID_DATA;
  if (n_streams == 0) return RPL_RESULT_OK;
  if (ans_type == 0x85 && (reinterpret_cast<uintptr_t>(capsules) & 3u) != 0) {
    c->err = "dense capsule buffer must be 4-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  rpl::CapsuleDecodeArgs a{};
  a.capsules = capsules;
  a.counts = capsule_counts;
  a.n_streams = n_streams;
  a.stride_capsules = stride_capsules;
  a.sample_duration_us = sample_duration_us;
  a.state_words = 2;
  a.state_in = state_in;
  a.nodes_out = reinterpret_cast<uint2*>(nodes_out);
  a.node_counts = node_counts;
  a.capsule_status = capsule_status;
  a.capsule_node_offset = capsule_node_offset;
  a.state_out = state_out;
  return decode_capsules_launch(c, ans_type, a, stream);
}

rpl_result rpl_decode_capsules(rpl_ctx* c, uint32_t ans_type, const uint8_t* capsules, uint32_t n_capsules,
                               uint32_t sample_duration_us, uint32_t* state, rpl_node_hq* nodes_out,
                               uint32_t* node_count, uint32_t* capsule_status, uint32_t* capsule_node_offset,
                               const rpl_timing* timing, const uint64_t* capsule_rx_us, uint64_t* node_ts_us) {
  if (!c || !node_count || (n_capsules && (!capsules || !nodes_out))) return RPL_RESULT_INVALID_DATA;
  const bool want_ts = timing || capsule_rx_us || node_ts_us;
  if (want_ts && !(timing && capsule_rx_us && node_ts_us)) {
    c->err = "timing, capsule_rx_us and node_ts_us go together";
    return RPL_RESULT_INVALID_DATA;
  }
  if (want_ts) sample_duration_us = timing->sample_duration_us;
  *node_count = 0;
  const uint32_t cbytes = capsule_bytes(c, ans_type), per = rpl_capsule_nodes(ans_type);
  if (cbytes == 0) return RPL_RESULT_INVALID_DATA;
  if (n_capsules == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, nullptr, &st)) return RPL_RESULT_OPERATION_FAIL;
  const size_t sb = (size_t)n_capsules * 4;
  // small: count, n_nodes, state in x2, state out x2
  struct Regions { uint8_t* caps; rpl_node_hq* nodes; uint32_t *status, *offsets, *small; uint64_t *rx, *ts; };
  auto layout = [&](Carve& k) {
    const size_t n = n_capsules, ts = want_ts ? n : 0;
    return Regions{k.take<uint8_t>(n * cbytes), k.take<rpl_node_hq>(n * per), k.take<uint32_t>(n), k.take<uint32_t>(n),
                   k.take<uint32_t>(8), k.take<uint64_t>(ts), k.take<uint64_t>(ts * per)};
  };
  if (const rpl_result r = grow_stage(c, 1, layout); r != RPL_RESULT_OK) return r;
  Carve k{c->lane[0].stage};
  const Regions d = layout(k);
  uint32_t small[8] = {n_capsules, 0u, state ? state[0] : 0u, state ? state[1] : 0u, 0u, 0u, 0u, 0u};
  RPL_CUDA(c, cudaMemcpyAsync(d.caps, capsules, (size_t)n_capsules * cbytes, cudaMemcpyHostToDevice, st),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(d.small, small, 32, cudaMemcpyHostToDevice, st), RPL_RESULT_OPERATION_FAIL);
  rpl_result r = rpl_decode_capsules_batch_dev(c, ans_type, d.caps, d.small, 1, n_capsules, sample_duration_us,
                                               d.small + 2, d.nodes, d.small + 1, d.status, d.offsets, d.small + 4, st);
  if (r != RPL_RESULT_OK) return r;
  if (want_ts) {
    RPL_CUDA(c, cudaMemcpyAsync(d.rx, capsule_rx_us, (size_t)n_capsules * 8, cudaMemcpyHostToDevice, st),
             RPL_RESULT_OPERATION_FAIL);
    r = rpl_node_timestamps_dev(c, ans_type, timing, d.rx, d.status, d.offsets, d.small, 1, n_capsules, d.ts, st);
    if (r != RPL_RESULT_OK) return r;
  }
  RPL_CUDA(c, cudaMemcpyAsync(small, d.small, 32, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  *node_count = small[1];
  if (state) {
    state[0] = small[4];
    state[1] = small[5];
  }
  if (want_ts)
    RPL_CUDA(c, cudaMemcpy(node_ts_us, d.ts, (size_t)small[1] * 8, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpy(nodes_out, d.nodes, (size_t)small[1] * 8, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  if (capsule_status)
    RPL_CUDA(c, cudaMemcpy(capsule_status, d.status, sb, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  if (capsule_node_offset)
    RPL_CUDA(c, cudaMemcpy(capsule_node_offset, d.offsets, sb, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_frame_capsules_dev(rpl_ctx* c, uint32_t ans_type, const uint8_t* bytes, const uint32_t* byte_counts,
                                  uint32_t n_streams, uint32_t stride_bytes, uint8_t* capsules_out,
                                  uint32_t stride_capsules, uint32_t* capsule_counts_out, uint32_t* bytes_left_out,
                                  void* stream) {
  if (!c || !bytes || !byte_counts || !capsules_out || !capsule_counts_out) return RPL_RESULT_INVALID_DATA;
  const uint32_t cb = rpl_capsule_bytes(ans_type);
  if (cb == 0 || ans_type == 0x83) {
    c->err = "byte-level framing serves the capsule formats with sync nibbles: 0x82, 0x84, 0x85, 0x86";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_streams == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::FrameArgs a{};
  a.bytes = bytes;
  a.byte_counts = byte_counts;
  a.n_streams = n_streams;
  a.stride_bytes = stride_bytes;
  a.capsule_bytes = cb;
  a.capsules_out = capsules_out;
  a.stride_capsules = stride_capsules;
  a.capsule_counts_out = capsule_counts_out;
  a.bytes_left_out = bytes_left_out;
  const int grid = (int)std::min<uint32_t>(n_streams, (uint32_t)c->num_sms * 8u);
  RPL_CUDA(c, rpl::launch_frame_capsules(a, grid, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

rpl_result rpl_decode_normal_batch_dev(rpl_ctx* c, const uint8_t* bytes, const uint32_t* byte_counts,
                                       uint32_t n_streams, uint32_t stride_bytes, rpl_node_hq* nodes_out,
                                       uint32_t* node_counts, uint32_t* fsm_state_out, uint32_t* node_end,
                                       void* stream) {
  if (!c || !bytes || !byte_counts || !nodes_out) return RPL_RESULT_INVALID_DATA;
  if (misaligned8(nodes_out)) {
    c->err = "nodes_out must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_streams == 0) return RPL_RESULT_OK;
  rpl::NormalDecodeArgs a{};
  a.bytes = bytes;
  a.byte_counts = byte_counts;
  a.n_streams = n_streams;
  a.stride_bytes = stride_bytes;
  a.nodes_out = reinterpret_cast<uint2*>(nodes_out);
  a.node_counts = node_counts;
  a.fsm_state_out = fsm_state_out;
  a.node_end = node_end;
  return decode_normal_launch(c, a, stream);
}

rpl_result rpl_decode_normal(rpl_ctx* c, const uint8_t* bytes, uint32_t n_bytes, rpl_node_hq* nodes_out,
                             uint32_t* node_count) {
  if (!c || !node_count || (n_bytes && (!bytes || !nodes_out))) return RPL_RESULT_INVALID_DATA;
  *node_count = 0;
  if (n_bytes < 5) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, nullptr, &st)) return RPL_RESULT_OPERATION_FAIL;
  struct Regions { uint8_t* bytes; rpl_node_hq* nodes; uint32_t* small; };  // small: byte count, node count
  auto layout = [&](Carve& k) {
    return Regions{k.take<uint8_t>(n_bytes), k.take<rpl_node_hq>(n_bytes / 5), k.take<uint32_t>(2)};
  };
  if (const rpl_result r = grow_stage(c, 1, layout); r != RPL_RESULT_OK) return r;
  Carve k{c->lane[0].stage};
  const Regions d = layout(k);
  uint32_t small[2] = {n_bytes, 0u};
  RPL_CUDA(c, cudaMemcpyAsync(d.bytes, bytes, n_bytes, cudaMemcpyHostToDevice, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(d.small, small, 8, cudaMemcpyHostToDevice, st), RPL_RESULT_OPERATION_FAIL);
  const rpl_result r =
      rpl_decode_normal_batch_dev(c, d.bytes, d.small, 1, n_bytes, d.nodes, d.small + 1, nullptr, nullptr, st);
  if (r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaMemcpyAsync(small, d.small, 8, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  *node_count = small[1];
  RPL_CUDA(c, cudaMemcpy(nodes_out, d.nodes, (size_t)small[1] * 8, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

// ---- scan assembly (SURVEY.md 8(f) rank 2) ------------------------------------------------------
}  // extern "C"

namespace {
// copy mode (scans_out) or view mode (views_out + writable nodes); with `list` (a mixed byte session's launch over the
// n_streams streams of one answer type) the regions are those of the list_span streams of the chunk
rpl_result assemble_common(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* node_counts,
                                  uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                  const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                  uint32_t stride_capsules, uint32_t max_nodes, uint32_t max_scans,
                                  uint32_t scan_stride, rpl_node_hq* scans_out, rpl_scan_view* views_out, uint32_t* scan_len,
                                  uint32_t* scans_per_stream, const uint64_t* node_ts_us,
                                  uint64_t* scan_begin_ts_us, void* stream, const uint32_t* scan_starts = nullptr,
                                  uint32_t starts_stride = 0, const uint32_t* scan_start_counts = nullptr,
                                  const uint32_t* carry_len = nullptr, rpl_node_hq* carry_out = nullptr,
                                  uint32_t* carry_len_out = nullptr, const rpl::AssembleStampArgs* stamp = nullptr,
                                  rpl::StreamCounters* counters = nullptr, uint32_t counted_capsule_bytes = 0,
                                  const rpl::StreamList* list = nullptr, uint32_t list_span = 0) {
  if (!c || !nodes || !node_counts || (!scans_out && !views_out) || !scan_len || !scans_per_stream) return RPL_RESULT_INVALID_DATA;
  const uint32_t span = list ? list_span : n_streams;
  if (views_out && (unsigned long long)span * stride_nodes > 0xFFFFFFFFull) {
    c->err = "view mode addresses nodes with 32 bits: n_streams * stride_nodes must stay below 2^32";
    return RPL_RESULT_INVALID_DATA;
  }
  const bool any = capsule_status || capsule_node_offset || capsule_counts;
  if (any && !(capsule_status && capsule_node_offset && capsule_counts)) {
    c->err = "capsule_status, capsule_node_offset and capsule_counts go together";
    return RPL_RESULT_INVALID_DATA;
  }
  if (max_nodes == 0 || max_scans == 0 || scan_stride < max_nodes) {
    c->err = "need max_nodes > 0, max_scans > 0, scan_stride >= max_nodes";
    return RPL_RESULT_INVALID_DATA;
  }
  if (misaligned8(nodes) || misaligned8(scans_out) || misaligned8(node_ts_us) || misaligned8(scan_begin_ts_us)) {
    c->err = "node and timestamp buffers must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_streams == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  const size_t need_rp = (size_t)span * std::max<uint32_t>(stride_capsules, 1u);
  const size_t need_desc = (size_t)span * max_scans;
  if (need_rp > c->reset_prefix_cap) {
    cudaFree(c->d_reset_prefix);
    c->d_reset_prefix = nullptr;
    RPL_CUDA(c, dev_alloc(&c->d_reset_prefix, need_rp), RPL_RESULT_INSUFFICIENT_MEMORY);
    c->reset_prefix_cap = need_rp;
  }
  if (need_desc > c->desc_cap) {
    cudaFree(c->d_desc);
    c->d_desc = nullptr;
    RPL_CUDA(c, dev_alloc(&c->d_desc, need_desc), RPL_RESULT_INSUFFICIENT_MEMORY);
    c->desc_cap = need_desc;
  }
  rpl::AssembleArgs a{};
  a.nodes = reinterpret_cast<const uint2*>(nodes);
  a.node_counts = node_counts;
  a.n_streams = n_streams;
  a.stride_nodes = stride_nodes;
  a.capsule_status = capsule_status;
  a.capsule_node_offset = capsule_node_offset;
  a.capsule_counts = capsule_counts;
  a.stride_capsules = std::max<uint32_t>(stride_capsules, 1u);
  a.max_nodes = max_nodes;
  a.max_scans = max_scans;
  a.scan_stride = scan_stride;
  a.scans_out = reinterpret_cast<uint2*>(scans_out);
  a.views_out = reinterpret_cast<uint2*>(views_out);
  a.nodes_mut = views_out ? reinterpret_cast<uint2*>(const_cast<rpl_node_hq*>(nodes)) : nullptr;
  a.scan_len = scan_len;
  a.scans_per_stream = scans_per_stream;
  a.node_ts_us = reinterpret_cast<const unsigned long long*>(node_ts_us);
  a.scan_begin_ts_us = reinterpret_cast<unsigned long long*>(scan_begin_ts_us);
  a.scan_starts = scan_starts;
  a.scan_start_counts = scan_start_counts;
  a.starts_stride = starts_stride;
  a.reset_prefix = c->d_reset_prefix;
  a.desc = c->d_desc;
  a.carry_len = carry_len;
  a.carry_out = reinterpret_cast<uint2*>(carry_out);
  a.carry_len_out = carry_len_out;
  a.counters = counters;
  a.counted_capsule_bytes = counted_capsule_bytes;
  const int grid = (int)std::min<uint32_t>(n_streams, (uint32_t)c->num_sms * 4u);
  if (stamp)
    RPL_CUDA(c, rpl::launch_assemble_stamped(a, *stamp, grid, st, list), RPL_RESULT_OPERATION_FAIL);
  else
    RPL_CUDA(c, rpl::launch_assemble(a, grid, st, list), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}
}  // namespace

extern "C" {

rpl_result rpl_assemble_scans_dev(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* node_counts,
                                  uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                  const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                  uint32_t stride_capsules, uint32_t max_nodes, uint32_t max_scans,
                                  uint32_t scan_stride, rpl_node_hq* scans_out, uint32_t* scan_len,
                                  uint32_t* scans_per_stream, const uint64_t* node_ts_us,
                                  uint64_t* scan_begin_ts_us, void* stream) {
  if (!scans_out) return RPL_RESULT_INVALID_DATA;
  return assemble_common(c, nodes, node_counts, n_streams, stride_nodes, capsule_status, capsule_node_offset,
                         capsule_counts, stride_capsules, max_nodes, max_scans, scan_stride, scans_out, nullptr, scan_len,
                         scans_per_stream, node_ts_us, scan_begin_ts_us, stream);
}

rpl_result rpl_assemble_scan_views_dev(rpl_ctx* c, rpl_node_hq* nodes, const uint32_t* node_counts,
                                       uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                       const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                       uint32_t stride_capsules, uint32_t max_nodes, uint32_t max_scans,
                                       rpl_scan_view* views_out, uint32_t* scan_len, uint32_t* scans_per_stream,
                                       const uint64_t* node_ts_us, uint64_t* scan_begin_ts_us, void* stream) {
  if (!views_out) return RPL_RESULT_INVALID_DATA;
  return assemble_common(c, nodes, node_counts, n_streams, stride_nodes, capsule_status, capsule_node_offset,
                         capsule_counts, stride_capsules, max_nodes, max_scans, max_nodes, nullptr, views_out, scan_len,
                         scans_per_stream, node_ts_us, scan_begin_ts_us, stream);
}

rpl_result rpl_assemble_scan_views_starts_dev(rpl_ctx* c, rpl_node_hq* nodes, const uint32_t* node_counts,
                                              uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                              const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                              uint32_t stride_capsules, const uint32_t* scan_starts,
                                              uint32_t starts_stride, const uint32_t* scan_start_counts,
                                              uint32_t max_nodes, uint32_t max_scans, rpl_scan_view* views_out,
                                              uint32_t* scan_len, uint32_t* scans_per_stream, const uint64_t* node_ts_us,
                                              uint64_t* scan_begin_ts_us, void* stream) {
  if (!views_out || !scan_starts || !scan_start_counts || starts_stride == 0) return RPL_RESULT_INVALID_DATA;
  return assemble_common(c, nodes, node_counts, n_streams, stride_nodes, capsule_status, capsule_node_offset,
                         capsule_counts, stride_capsules, max_nodes, max_scans, max_nodes, nullptr, views_out, scan_len,
                         scans_per_stream, node_ts_us, scan_begin_ts_us, stream, scan_starts, starts_stride,
                         scan_start_counts);
}

rpl_result rpl_scan_views_dev(rpl_ctx* c, const rpl_node_hq* nodes, uint64_t nodes_total, const rpl_scan_view* views,
                              uint32_t n_scans, uint32_t stride, const rpl_scan_params* params, rpl_node_hq* nodes_out,
                              float* ranges, float* intensities, uint32_t* beam_counts, float* angle_increment,
                              uint32_t* status, uint32_t* path, void* stream) {
  if (!c || !views || !nodes || !params) return RPL_RESULT_INVALID_DATA;
  if (!rpl::scan_small_applies(stride) || (params->flags & RPL_FLAG_NO_SMALL)) {
    c->err = "scan views are served by the shared-memory kernels: stride (the longest scan) must be <= 8192 nodes";
    return RPL_RESULT_INVALID_DATA;
  }
  if ((reinterpret_cast<uintptr_t>(nodes) & 15u) != 0) {
    c->err = "the node buffer of a view batch must be 16-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  return enqueue_scan(c, c->lane[0], nodes, reinterpret_cast<const uint32_t*>(views), n_scans, stride, params, nodes_out,
                      ranges, intensities, beam_counts, angle_increment, status, path, st,
                      reinterpret_cast<const uint2*>(views), nodes_total);
}

}  // extern "C"

// ---- capsule stream session (DESIGN.md 5.7) ------------------------------------------------------------------------
// Per stream: the held capsule with the decoder's cross-capsule state (one rpl::kHeldWords record; HQ capsules hold
// nothing), and the revolution left open, kept in front of the next push's nodes so that a scan spanning pushes is one
// contiguous view.  Each stream's region of an arena is [max_nodes carry slots][nodes per capsule * stride_capsules new
// nodes]; push t decodes into arena t % 2 and its assembler writes the new open revolution into the carry slots of the
// other arena, because the scans push t closes are read from this arena's carry slots by the scan kernels after the
// assembler.
// A stamped push (rpl_capsule_stream_push*_ts*) runs the stamped decoder (0x81) and assembler instead; they keep,
// beside the carry, the open revolution's stamp (open_ts, per arena like carry_len) and, for express and ultra, the
// held capsule's receive time (held_rx).  An unstamped push leaves both stale, so the next stamped push counts them as
// unknown (carry_stamped false); an import folds that into every stream's own values first, open_ts 0 and held_rx
// kRxUnknown, since the stream it writes keeps the stamps its record carries.
// A byte session (rpl_capsule_stream_create_bytes) takes the raw bytes of the serial stream instead of framed capsules.
// On a capsule answer type each push is framed first (frame.cu's session instantiation, the search carried in the
// framer record) into the session's own capsule slots, which the decoder then reads as a framed session's push;
// stride_capsules counts those slots, and a stamped push's capsule receive times come out of the framer.  On 0x81
// standard nodes the decoder reads the pushed bytes itself: the held record keeps the byte machine, stride_capsules
// counts bytes (cap_bytes 1), and there are no capsule reports (the standard unpacker requests no scan resets).
struct rpl_capsule_stream {
  rpl_ctx* c = nullptr;
  uint32_t ans_type = 0, cap_bytes = 0;    // answer type, bytes per capsule (0x81: 1)
  uint32_t n_streams = 0, stride_capsules = 0, max_nodes = 0, max_scans = 0;  // stride_capsules: 0x81, bytes
  // what a push takes, fixed at create: bytes (a byte session) or framed capsules; per stream at most stride_in of
  // them (bytes or capsules), in_stream bytes of input
  bool bytes = false;
  uint32_t stride_in = 0;
  size_t in_stream = 0;
  uint32_t stride_nodes = 0, starts_stride = 0;
  uint32_t chunk_dev = 0, chunk_host = 0;  // streams per scan launch (context's max_scans), per host-push chunk
  uint32_t parity = 0;                     // arena of the next push
  rpl_node_hq* arena[2] = {nullptr, nullptr};
  uint32_t* carry_len[2] = {nullptr, nullptr};  // [n_streams] open revolution in front of arena[p]'s new nodes
  uint32_t* held = nullptr;                     // [n_streams][kHeldWords]
  uint32_t *status = nullptr, *offsets = nullptr, *node_counts = nullptr;  // status, offsets: capsule formats only
  uint32_t *starts = nullptr, *start_counts = nullptr;  // dense only: the decoder's scan-start list
  uint32_t* scan_len = nullptr;
  rpl_scan_view* views = nullptr;
  cudaEvent_t done = nullptr;                   // the last push_dev: later calls on other streams wait for it
  unsigned long long* open_ts[2] = {nullptr, nullptr};  // [n_streams] stamp of the open revolution (0: unknown)
  unsigned long long* held_rx = nullptr;        // [n_streams] express, ultra: receive time of the held capsule
  uint32_t* scan_ends = nullptr;                // 0x81: [n_streams][new nodes] end bytes of the scan-start records
  bool prev_stamped = true;                     // the last push had receive times (a fresh session holds nothing)
  bool carry_stamped = true;                    // open_ts[parity] and held_rx hold every stream's stamps (else none)
  // a byte session of a capsule answer type (else null): the framer records, this push's framed capsules
  uint32_t* framer = nullptr;                   // [n_streams][kFramerWords]
  uint8_t* framed = nullptr;                    // [n_streams][stride_capsules][cap_bytes]
  uint32_t* framed_counts = nullptr;            // [n_streams]
  unsigned long long* framed_rx = nullptr;      // [n_streams][stride_capsules] (stamped pushes)
  size_t framed_stride = 0;                     // bytes per stream of `framed`
  // a mixed byte session (rpl_capsule_stream_create_bytes_mixed; ans_type 0): each stream's answer type, and for the
  // host-push chunks (0) and the device-push chunks (1) the chunk-relative indices of every chunk's streams grouped by
  // answer type (lists[k] + s0: the chunk from stream s0's), which list_begin[k] directs: entry 7 * chunk + t the first
  // position of type 0x81 + t in that chunk's list (t = 6: its end)
  std::vector<uint32_t> types;                  // [n_streams] host; empty: a single-type session
  uint32_t* lists[2] = {nullptr, nullptr};     // [n_streams] device
  std::vector<uint32_t> list_begin[2];
  // the last push, as the cloud calls replay it: its views count from the first stream of their chunk
  uint32_t cloud_chunk = 0;                     // streams per chunk (chunk_host or chunk_dev); 0: no push, or it failed
  uint32_t cloud_arena = 0;                     // the arena its views point into
  // the messages of the last push (rpl_capsule_stream_*_msgs*): a stamped push's slot stamps, the per-stream settings
  unsigned long long* slot_begin = nullptr;     // [n_streams * max_scans] scan-begin stamps (0: unused, unknown)
  unsigned long long* slot_end = nullptr;       // [n_streams * max_scans] the closing scan-start node's stamp
  rpl::StreamMsgHeader* msg_hdr = nullptr;      // [n_streams] device
  std::vector<rpl::StreamMsgHeader> msg_hdr_host;
  unsigned char* msg_work = nullptr;            // the scan kernels' outputs and the tables of a messages call
  size_t msg_work_bytes = 0;
  // the per-stream lidar settings (rpl_capsule_stream_set_lidars) that calls with RPL_FLAG_PER_STREAM /
  // RPL_CLOUD_PER_STREAM read; empty until the first call sets every stream
  rpl::LidarSettings* lidars = nullptr;         // [n_streams] device
  std::vector<rpl::LidarSettings> lidars_host;
  uint32_t lidar_modes = 0;                     // LidarTable::modes of the table
  // the per-stream clouds (rpl_capsule_stream_set_clouds) that calls with RPL_CLOUD_PER_STREAM_CHAIN read: the entries
  // as set (empty until the first call sets every stream), and the table resolved against the frames' range_max
  // (clouds_resolve): on the device, the routes present (bit per rpl::CloudRoute), the largest sor_k and whether a
  // voxel grid runs, and why a flagged call fails (empty: it does not)
  std::vector<rpl_cloud_settings> clouds_host;
  rpl::CloudSettings* clouds = nullptr;         // [n_streams] device
  uint32_t cloud_routes = 0, cloud_sor_k = 0;
  // the same table for calls with RPL_CLOUD_PER_STREAM_FOOTPRINTS: a stream with footprint polygons takes the separate
  // passes where it would have been fused, so that the footprint pass runs between xyz and SOR (clouds_resolve)
  rpl::CloudSettings* clouds_fp = nullptr;      // [n_streams] device
  uint32_t cloud_routes_fp = 0;
  bool cloud_voxel = false;
  std::string clouds_bad;
  // the per-stream LaserScan filters (rpl_capsule_stream_set_scan_filters) that calls with RPL_FLAG_PER_STREAM_FILTERS
  // read: the entries as set (empty until the first call sets every stream) and as the kernel reads them
  std::vector<rpl_scan_filter_settings> filters_host;
  rpl::ScanFilter* filters = nullptr;           // [n_streams] device
  // their footprints (rpl_capsule_stream_set_scan_footprints): as set (empty until the first call sets every stream)
  // and as the kernel reads them (nullptr until then: no stream has a footprint)
  std::vector<rpl_scan_footprint> footprints_host;
  rpl::ScanFootprint* footprints = nullptr;     // [n_streams] device
  // the transforms of the projected clouds (rpl_capsule_stream_set_scan_cloud_transforms) that calls with
  // RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS read: the entries and target frames as set (empty until the first call sets
  // every stream), their rows (scan_cloud_rows) and each stream's resolved message header -- the target frame's, a
  // disabled entry's the LaserScan's -- rebuilt by set_frames as well (transforms_resolve)
  std::vector<rpl_scan_cloud_transform> xf_host;
  std::vector<std::string> xf_frames;
  float4* xf = nullptr;                         // [n_streams][3] device
  rpl::StreamMsgHeader* xf_hdr = nullptr;       // [n_streams] device
  std::vector<rpl::StreamMsgHeader> xf_hdr_host;
  // the re-gridded scans' entries (rpl_capsule_stream_set_rescans) as set (empty until the first call sets every
  // stream), as rescan_kernel reads them, and their ranges_size (0: disabled), which sizes the messages
  std::vector<rpl_rescan_settings> rescan_host;
  rpl::RescanGrid* rescan = nullptr;            // [n_streams] device
  uint32_t* rescan_bins = nullptr;              // [n_streams] device
  // the windows over them (rpl_capsule_stream_set_rescan_windows): the entries as set (empty until the first call: every
  // stream's observations is 1) and, laid out from both tables by either set call (windows_layout), each stream's
  // window as the kernel reads it, its {count, head}, the ring, and the enabled streams with a window (ascending)
  std::vector<rpl_rescan_window> win_host;
  rpl::RescanWindow* win = nullptr;             // [n_streams] device
  uint2* win_state = nullptr;                   // [n_streams] device, zeroed at the first call
  float* win_ring = nullptr;
  uint32_t* win_streams = nullptr;              // [n_streams] device, win_streams_host.size() used
  std::vector<uint32_t> win_streams_host;
  std::vector<rpl::RescanWindow> win_layout_host;  // as win
  // the groups merged into one scan each (rpl_capsule_stream_set_rescan_merges; mg_set false until the first call), in
  // one device block (MergeTables): each group's members ascending by group (mg_begin), the grouped streams ascending
  // (mg_streams_host; a chunk's hold launch takes its run of them), and the merge pushes that succeeded (mg_seq).  The
  // host form stages its merged messages and their directory in mg_stage.
  bool mg_set = false;
  uint32_t mg_groups = 0, mg_seq = 0;
  std::vector<uint32_t> mg_members_host, mg_begin_host, mg_streams_host;
  unsigned char* mg_block = nullptr;
  unsigned char* mg_stage = nullptr;
  size_t mg_stage_bytes = 0;
  unsigned char* node_work = nullptr;           // the tables of a nodes call (NodeWork)
  // [n_streams] device, zeroed at create: what every push decoded and lost (rpl_capsule_stream_counters); a stream's
  // record is written by the one CTA of each kernel that serves the stream
  rpl::StreamCounters* counters = nullptr;
  // message pushes (rpl_capsule_stream_push_{laserscan,cloud}_msgs*), made by the first: the device tables of the push's
  // slots (PushMsgWork), the host form's pinned read-back of each lane's chunk's extent ([kLanes][3]) with the events
  // that tell it is there, and the event that orders the chunks' directories
  unsigned char* push_msg_work = nullptr;
  unsigned long long* push_msg_extent = nullptr;
  cudaEvent_t push_msg_extent_ready[kLanes] = {}, push_msg_dir_order = nullptr;
  // pushes that also project their LaserScans (rpl_capsule_stream_push_scan_cloud_msgs*), made by the first: the
  // clouds' directory carry and every slot's kept count (ScanCloudWork), the host form's pinned read-back of each
  // lane's chunk's cloud extent ([kLanes][3]; push_msg_extent_ready tells it is there) and the order of the chunks'
  // cloud directories
  unsigned char* push_scan_cloud_work = nullptr;
  unsigned long long* push_scan_cloud_extent = nullptr;
  cudaEvent_t push_scan_cloud_dir_order = nullptr;
  // export / import (rpl_capsule_stream_export, _import): the device staging of the records and their tables
  unsigned char* migrate_work = nullptr;
  size_t migrate_work_bytes = 0;
};

static_assert(sizeof(rpl::StreamCounters) == sizeof(rpl_stream_counters) &&
                  offsetof(rpl::StreamCounters, bytes_in) == offsetof(rpl_stream_counters, bytes_in) &&
                  offsetof(rpl::StreamCounters, skipped_bytes) == offsetof(rpl_stream_counters, skipped_bytes) &&
                  offsetof(rpl::StreamCounters, scan_resets) == offsetof(rpl_stream_counters, scan_resets) &&
                  offsetof(rpl::StreamCounters, nodes) == offsetof(rpl_stream_counters, nodes) &&
                  offsetof(rpl::StreamCounters, scans_rewound) == offsetof(rpl_stream_counters, scans_rewound) &&
                  offsetof(rpl::StreamCounters, scans_unreturned) == offsetof(rpl_stream_counters, scans_unreturned),
              "rpl::StreamCounters must be rpl_stream_counters byte for byte");

static_assert(sizeof(rpl::LidarSettings) == sizeof(rpl_lidar_settings) &&
                  offsetof(rpl::LidarSettings, mode_a) == offsetof(rpl_lidar_settings, scan_processing) &&
                  offsetof(rpl::LidarSettings, inverted) == offsetof(rpl_lidar_settings, inverted) &&
                  offsetof(rpl::LidarSettings, timing) == offsetof(rpl_lidar_settings, timing) &&
                  sizeof(rpl::TimingDesc) == sizeof(rpl_timing),
              "rpl::LidarSettings must be rpl_lidar_settings byte for byte");

static_assert(sizeof(rpl::CloudSettings) == sizeof(rpl_cloud_settings) &&
                  offsetof(rpl::CloudSettings, voxel) == offsetof(rpl_cloud_settings, voxel_size) &&
                  offsetof(rpl::CloudSettings, sor_k) == offsetof(rpl_cloud_settings, sor_k) &&
                  offsetof(rpl::CloudSettings, sor_alpha) == offsetof(rpl_cloud_settings, sor_alpha) &&
                  offsetof(rpl::CloudSettings, route) == offsetof(rpl_cloud_settings, enabled) &&
                  offsetof(rpl_cloud_settings, sor_alpha) == offsetof(rpl_cloud_params, sor_alpha),
              "rpl::CloudSettings must be laid out as rpl_cloud_settings, and its first 24 bytes as rpl_cloud_params");

namespace {

// a stamped push's receive times and stamp output (rx, scan_ts: of the first stream of the call they are passed to)
struct StampPush {
  rpl::TimingDesc timing;
  const unsigned long long* rx;         // capsule_rx_us [.][stride_capsules], byte pushes: chunk_rx_us [.][stride_chunks]
  uint32_t chunk_bytes, stride_chunks;  // a framed push's chunk_bytes is 1; stride_chunks: ceil(stride_in / chunk_bytes)
  unsigned long long* scan_ts;          // scan_begin_ts_us [.][max_scans]
};

// A cloud call's per-stream chains (RPL_CLOUD_PER_STREAM_CHAIN): the session's resolved table at the chunk's first
// stream (nullptr before the first set_clouds) and what the whole table holds
struct CloudChains {
  const rpl::CloudSettings* at;
  uint32_t routes;  // bit r: some stream has rpl::CloudRoute r
  uint32_t sor_k;   // the largest sor_k of the streams with SOR
  bool voxel;       // some stream has a voxel grid
};

// the per-stream chains from stream s0 on (at: nullptr before the first set_clouds); fp: the table of a chunk that runs
// the footprint pass
CloudChains chains_at(const rpl_capsule_stream* cs, uint32_t s0, bool fp = false) {
  if (fp) return CloudChains{cs->clouds ? cs->clouds_fp + s0 : nullptr, cs->cloud_routes_fp, cs->cloud_sor_k, cs->cloud_voxel};
  return CloudChains{cs->clouds ? cs->clouds + s0 : nullptr, cs->cloud_routes, cs->cloud_sor_k, cs->cloud_voxel};
}

// a footprint with at least one polygon
bool has_polygons(const rpl_scan_footprint& e) {
  for (uint32_t n : e.n_vertices)
    if (n != 0) return true;
  return false;
}

// the footprints of a cloud call with RPL_CLOUD_PER_STREAM_FOOTPRINTS over streams [s0, s0 + ns): the table at s0, or
// nullptr when the call has no flag or no stream of the range has a polygon (no footprint pass)
const rpl::ScanFootprint* cloud_footprints_at(const rpl_capsule_stream* cs, const rpl_cloud_params* p, uint32_t s0,
                                              uint32_t ns) {
  if (!p || (p->flags & RPL_CLOUD_PER_STREAM_FOOTPRINTS) == 0 || cs->footprints_host.empty()) return nullptr;
  const uint32_t e = std::min(cs->n_streams, s0 + ns);
  for (uint32_t s = s0; s < e; ++s)
    if (has_polygons(cs->footprints_host[s])) return cs->footprints + s0;
  return nullptr;
}

// Where a chunk of streams lives on the device between the kernels of capsule_stream_chunk, every pointer at the
// chunk's first stream.  A session's chunk decodes behind node_first carry slots per stream (node_stride != 0),
// keeps the held record and hands the open revolution to the other arena.  The chain's has no held record, no carry
// and node_stride 0, so that the decoder and the assembler run their stateless kernels.
struct WireChunk {
  uint32_t ans_type, stride_capsules, max_nodes, max_scans, starts_stride;
  uint32_t stride_nodes;             // each stream's region of `nodes`
  uint32_t node_stride, node_first;  // the decoder's: a session's stride_nodes and max_nodes; 0, 0 for the chain
  rpl_node_hq *nodes, *carry_out;
  uint32_t *node_counts, *scan_len, *held, *carry_len_out;
  const uint32_t* carry_len;
  uint32_t *status, *offsets;       // capsule formats only: the per-capsule reports (scan-reset requests)
  uint32_t *starts, *start_counts;  // dense only: the decoder's scan-start list (others: the assembler's flag pass)
  rpl_scan_view* views;
  // a stamped session push's: 0x81 scan-start record ends, the open revolution's stamp, the held capsule's rx
  uint32_t* node_end;
  unsigned long long *open_ts_in, *open_ts_out, *held_rx;
  unsigned long long *slot_begin, *slot_end;
  bool prev_stamped;
  // a byte session's: the input is raw bytes [.][stride_bytes], framed into `framed` first
  uint32_t stride_bytes;
  uint32_t *framer, *framed_counts;
  uint8_t* framed;
  unsigned long long* framed_rx;
  size_t framed_stride;
  // a mixed byte session's: the chunk's streams by answer type (the session's lists and list_begin at this chunk)
  const uint32_t* lists;
  const uint32_t* list_begin;
  // a session push with RPL_FLAG_PER_STREAM: the chunk's first stream's entry of the session's table (else nullptr)
  const rpl::LidarSettings* lidars;
  uint32_t lidar_modes;
  // a session's counters (the chain's: nullptr); a framed session's bytes per capsule, which the assembler counts in
  // (a byte session's framer or 0x81 decoder counts the bytes)
  rpl::StreamCounters* counters;
  uint32_t counted_capsule_bytes;
  // the session's per-stream chains, which a PointCloud2 push with RPL_CLOUD_PER_STREAM_CHAIN reads, and with
  // RPL_CLOUD_PER_STREAM_FOOTPRINTS the chunk's first stream's footprint when some stream of the chunk has a polygon
  // (else nullptr: no footprint pass)
  CloudChains clouds;
  const rpl::ScanFootprint* cloud_footprints;
  // a LaserScan push with RPL_FLAG_PER_STREAM_FILTERS: the chunk's first stream's entry of the session's filters, when
  // some stream of the chunk has its filters enabled (else nullptr: no filter launch)
  const rpl::ScanFilter* filters;
  const rpl::ScanFootprint* footprints;  // with filters: the chunk's first stream's footprint (nullptr: none)
};

// the filters of a call with RPL_FLAG_PER_STREAM_FILTERS over streams [s0, s0 + ns): the table at s0, or nullptr when
// the call has no flag or no stream of the range is enabled
const rpl::ScanFilter* filters_at(const rpl_capsule_stream* cs, const rpl_scan_params* p, uint32_t s0, uint32_t ns) {
  if ((p->flags & RPL_FLAG_PER_STREAM_FILTERS) == 0 || cs->filters_host.empty()) return nullptr;
  const uint32_t e = std::min(cs->n_streams, s0 + ns);
  for (uint32_t s = s0; s < e; ++s)
    if (cs->filters_host[s].enabled) return cs->filters + s0;
  return nullptr;
}

// the footprints of stream s0 on (nullptr before the first set_scan_footprints)
const rpl::ScanFootprint* footprints_at(const rpl_capsule_stream* cs, uint32_t s0) {
  return cs->footprints ? cs->footprints + s0 : nullptr;
}

// the filters at `filters` with the footprints at `footprints` (nullptr: none) over n scan slots, per slots per entry:
// rows (ranges / intens at stride) or, with msg_out, the placed messages of `place`; beams and inc the scan kernels'
// beam counts and angle increments of the slots
rpl_result filter_scans(rpl_ctx* c, const rpl::ScanFilter* filters, const rpl::ScanFootprint* footprints, uint32_t per,
                        uint32_t n, float* ranges, const float* intens, uint32_t stride, uint8_t* msg_out,
                        const unsigned long long* place, const uint32_t* beams, const float* inc, cudaStream_t st) {
  rpl::ScanFilterArgs a{};
  a.filters = filters;
  a.footprints = footprints;
  a.per_filter = per;
  a.ranges = ranges;
  a.intensities = intens;
  a.stride = stride;
  a.msg_out = msg_out;
  a.place = place;
  a.beam_counts = beams;
  a.angle_increment = inc;
  a.n_scans = n;
  RPL_CUDA(c, rpl::launch_scan_filter(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// session cs's chunk from stream s0 in the push under way (arena cs->parity) with params' flags (RPL_FLAG_PER_STREAM,
// RPL_FLAG_PER_STREAM_FILTERS) and a PointCloud2 push's cloud params (nullable); dev: a device push's chunking (else a
// host push's)
WireChunk session_chunk(const rpl_capsule_stream* cs, uint32_t s0, const rpl_scan_params* params, bool dev,
                        const rpl_cloud_params* cloud = nullptr) {
  const bool per_stream = (params->flags & RPL_FLAG_PER_STREAM) != 0;
  const uint32_t p = cs->parity, sc = cs->stride_capsules;
  const size_t sn = (size_t)s0 * cs->stride_nodes, so = (size_t)s0 * cs->max_scans;
  WireChunk w{};
  w.ans_type = cs->ans_type;
  w.stride_capsules = sc;
  w.max_nodes = cs->max_nodes;
  w.max_scans = cs->max_scans;
  w.stride_nodes = w.node_stride = cs->stride_nodes;
  w.node_first = cs->max_nodes;
  w.starts_stride = cs->starts_stride;
  w.nodes = cs->arena[p] + sn;
  w.node_counts = cs->node_counts + s0;
  w.status = cs->status ? cs->status + (size_t)s0 * sc : nullptr;
  w.offsets = cs->offsets ? cs->offsets + (size_t)s0 * sc : nullptr;
  w.starts = cs->starts ? cs->starts + (size_t)s0 * cs->starts_stride : nullptr;
  w.start_counts = cs->starts ? cs->start_counts + s0 : nullptr;
  w.views = cs->views + so;
  w.scan_len = cs->scan_len + so;
  w.held = cs->held + (size_t)s0 * rpl::kHeldWords;
  w.carry_len = cs->carry_len[p] + s0;
  w.carry_out = cs->arena[p ^ 1u] + sn;
  w.carry_len_out = cs->carry_len[p ^ 1u] + s0;
  w.node_end = cs->scan_ends ? cs->scan_ends + (size_t)s0 * (cs->stride_nodes - cs->max_nodes) : nullptr;
  w.open_ts_in = cs->open_ts[p] + s0;
  w.open_ts_out = cs->open_ts[p ^ 1u] + s0;
  w.held_rx = cs->held_rx + s0;
  w.slot_begin = cs->slot_begin + so;
  w.slot_end = cs->slot_end + so;
  w.prev_stamped = cs->carry_stamped;
  w.counters = cs->counters + s0;
  w.counted_capsule_bytes = cs->bytes ? 0u : cs->cap_bytes;
  if (cs->framer) {
    w.stride_bytes = cs->stride_in;
    w.framer = cs->framer + (size_t)s0 * rpl::kFramerWords;
    w.framed = cs->framed + (size_t)s0 * cs->framed_stride;
    w.framed_counts = cs->framed_counts + s0;
    w.framed_rx = cs->framed_rx + (size_t)s0 * sc;
    w.framed_stride = cs->framed_stride;
  }
  if (!cs->types.empty()) {
    const uint32_t chunk = dev ? cs->chunk_dev : cs->chunk_host;
    w.lists = cs->lists[dev] + s0;
    w.list_begin = cs->list_begin[dev].data() + (size_t)7 * (s0 / chunk);
  }
  if (per_stream) {
    w.lidars = cs->lidars + s0;
    w.lidar_modes = cs->lidar_modes;
  }
  w.cloud_footprints = cloud_footprints_at(cs, cloud, s0, dev ? cs->chunk_dev : cs->chunk_host);
  w.clouds = chains_at(cs, s0, w.cloud_footprints != nullptr);
  w.filters = filters_at(cs, params, s0, dev ? cs->chunk_dev : cs->chunk_host);
  w.footprints = w.filters ? footprints_at(cs, s0) : nullptr;
  return w;
}

// a mixed byte session's launch over the n streams of one answer type in a chunk
struct ListLaunch {
  rpl::StreamList l;
  uint32_t n;
};

// (frame ->) decode -> assemble of the ns streams of chunk w on `st` as answer type ans_type, or with `list` (a mixed
// byte session's) of the list->streams of that type alone; capsules / counts / sp as capsule_stream_chunk's
rpl_result decode_assemble(rpl_ctx* c, cudaStream_t st, const WireChunk& w, uint32_t ans_type, uint32_t ns,
                           const uint8_t* capsules, const uint32_t* counts, uint32_t sample_duration_us,
                           uint32_t* scans_per_stream, const StampPush* sp, const ListLaunch* list) {
  const uint32_t sc = w.stride_capsules, n = list ? list->n : ns;
  const bool normal = ans_type == RPL_ANS_MEASUREMENT;
  uint32_t* status = normal ? nullptr : w.status;  // the per-capsule reports
  uint32_t* offsets = normal ? nullptr : w.offsets;
  uint32_t* starts = ans_type == 0x85 ? w.starts : nullptr;
  uint32_t* start_counts = ans_type == 0x85 ? w.start_counts : nullptr;
  const rpl::StreamList* l = list ? &list->l : nullptr;
  uint32_t* ends = sp ? w.node_end : nullptr;
  StampPush framed_sp{};
  if (w.framer && !normal) {
    rpl::FrameArgs a{};
    a.bytes = capsules;
    a.byte_counts = counts;
    a.n_streams = n;
    a.stride_bytes = w.stride_bytes;
    a.capsule_bytes = rpl_capsule_bytes(ans_type);
    a.capsules_out = w.framed;
    a.stride_capsules = sc;
    a.capsule_counts_out = w.framed_counts;
    rpl::FrameStreamArgs f{};
    f.framer = w.framer;
    f.counters = w.counters;
    if (sp) {  // the framer turns the chunk receive times into the capsule receive times the assembler reads
      f.chunk_rx_us = sp->rx;
      f.chunk_bytes = sp->chunk_bytes;
      f.stride_chunks = sp->stride_chunks;
      f.capsule_rx_out = w.framed_rx;
      framed_sp = *sp;
      framed_sp.rx = w.framed_rx;
      sp = &framed_sp;
    }
    const int grid = (int)std::min<uint32_t>(n, (uint32_t)c->num_sms * 8u);
    RPL_CUDA(c, rpl::launch_frame_capsules_stream(a, f, grid, st, l), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
    capsules = w.framed;
    counts = w.framed_counts;
  }
  rpl_result r;
  if (normal) {
    rpl::NormalDecodeArgs a{};
    a.bytes = capsules;
    a.byte_counts = counts;
    a.n_streams = n;
    a.stride_bytes = list ? w.stride_bytes : sc;
    a.nodes_out = reinterpret_cast<uint2*>(w.nodes);
    a.node_counts = w.node_counts;
    a.held = w.held;
    a.node_stride = w.node_stride;
    a.node_first = w.node_first;
    a.node_end = ends;
    a.counters = w.counters;
    r = decode_normal_launch(c, a, st, l);
  } else {
    rpl::CapsuleDecodeArgs a{};
    a.capsules = capsules;
    a.counts = counts;
    a.n_streams = n;
    a.stride_capsules = sc;
    a.sample_duration_us = sample_duration_us;
    a.state_words = 1;
    a.nodes_out = reinterpret_cast<uint2*>(w.nodes);
    a.node_counts = w.node_counts;
    a.capsule_status = status;
    a.capsule_node_offset = offsets;
    a.scan_starts = starts;
    a.scan_start_counts = start_counts;
    a.starts_stride = w.starts_stride;
    a.held = w.held;
    a.node_stride = w.node_stride;
    a.node_first = w.node_first;
    a.lidars = w.lidars;
    r = decode_capsules_launch(c, ans_type, a, st, l);
  }
  if (r != RPL_RESULT_OK) return r;
  // the assembler's scratch belongs to the context: one assemble kernel at a time, whatever lane or stream
  if (!c->asm_done) RPL_CUDA(c, cudaEventCreateWithFlags(&c->asm_done, cudaEventDisableTiming), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamWaitEvent(st, c->asm_done, 0), RPL_RESULT_OPERATION_FAIL);
  rpl::AssembleStampArgs t{};
  if (sp) {
    t.ans_type = ans_type;
    t.timing = sp->timing;
    t.capsule_rx_us = status ? sp->rx : nullptr;
    t.node_end = ends;
    t.stride_ends = w.stride_nodes - w.node_first;
    t.chunk_bytes = sp->chunk_bytes;
    t.stride_chunks = sp->stride_chunks;
    t.chunk_rx_us = status ? nullptr : sp->rx;
    t.open_ts_in = w.open_ts_in;
    t.open_ts_out = w.open_ts_out;
    t.held_rx = w.held_rx;
    t.prev_stamped = w.prev_stamped ? 1u : 0u;
    t.slot_begin_us = w.slot_begin;
    t.slot_end_us = w.slot_end;
    t.lidars = w.lidars;
  }
  r = assemble_common(c, w.nodes, w.node_counts, n, w.stride_nodes, status, offsets, status ? counts : nullptr,
                      status ? sc : 0u, w.max_nodes, w.max_scans, w.max_nodes, nullptr, w.views, w.scan_len,
                      scans_per_stream, nullptr, sp ? reinterpret_cast<uint64_t*>(sp->scan_ts) : nullptr, st, starts,
                      starts ? w.starts_stride : 0u, start_counts, w.carry_len, w.carry_out, w.carry_len_out,
                      sp ? &t : nullptr, w.counters, w.counted_capsule_bytes, l, ns);
  if (r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaEventRecord(c->asm_done, st), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

// the footprint pass (cloud_footprint.cu) over the a.n_scans clouds of `a` (steps 1-3 done), scan s taking
// footprints[s / a.lidar_scans] (nullptr: `one`), mirrored where a.lidars says the stream is inverted
rpl_result footprint_clouds(rpl_ctx* c, const rpl::ScanBatchArgs& a, const rpl::ScanFootprint* footprints,
                            const rpl::ScanFootprint& one, uint32_t* point_counts, cudaStream_t st) {
  rpl::CloudFootprintArgs f{};
  f.xyzi = a.xyzi;
  f.point_counts = point_counts;
  f.n_scans = a.n_scans;
  f.stride = a.stride;
  f.footprints = footprints;
  f.lidars = a.lidars;
  f.per = a.lidar_scans ? a.lidar_scans : 1u;
  f.one = one;
  RPL_CUDA(c, rpl::launch_cloud_footprint(f, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// stream_cloud_chunk with RPL_CLOUD_PER_STREAM_CHAIN, `a` set up but for the table
rpl_result stream_chains_chunk(rpl_ctx* c, Lane& l, rpl::ScanBatchArgs a, const CloudChains& chains, bool separate,
                               const rpl::ScanFootprint* footprints, uint32_t* point_counts, cudaStream_t st) {
  using rpl::kCloudFused;
  using rpl::kCloudSeparate;
  using rpl::kCloudWindow;
  a.clouds = chains.at;
  // the fused kernel runs when the call may fuse (flags 0's rule: shared-memory kernels, a view longer than its arrays
  // handed on) and some stream is fusable; the window-only kernel for the other routes, and for the streams without a
  // cloud when the fused kernel does not run
  const bool fused = !separate && rpl::scan_small_applies(a.stride) &&
                     (rpl::scan_small_post_applies(a.stride) || a.views) && (chains.routes & (1u << kCloudFused)) != 0;
  const uint32_t separate_routes = (1u << kCloudSeparate) | (fused ? 0u : 1u << kCloudFused);
  a.cloud_launches = fused ? 2u : 0u;
  if (!fused || (chains.routes & ((1u << kCloudWindow) | separate_routes)) != 0) a.cloud_launches |= 1u;
  bool post_fused = false;
  rpl_result r = scratch_enter(c, l, st);
  if (r == RPL_RESULT_OK) r = enqueue_args(c, l, a, 0u, st, nullptr, &post_fused, true);
  if (r == RPL_RESULT_OK && footprints) r = footprint_clouds(c, a, footprints, rpl::ScanFootprint{}, point_counts, st);
  if (r != RPL_RESULT_OK) return r;
  const bool full = (chains.routes & separate_routes) != 0;  // the separate route's scans: every scan's pass
  if ((full || post_fused) && (chains.sor_k > 0 || chains.voxel)) {
    // (lane 0's cws and scratch, as below)
    Lane& post = c->lane[0];
    if (&l != &post && (r = scratch_enter(c, post, st)) != RPL_RESULT_OK) return r;
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 0 ? !full : !post_fused) continue;
      const rpl::CloudTable tab{chains.at, a.lidar_scans, a.cloud_launches, pass == 0 ? kCloudSeparate : kCloudFused};
      int launched = 0;
      RPL_CUDA(c, rpl::launch_cloud_post(a.xyzi, point_counts, a.n_scans, a.stride, chains.sor_k, 0.0f,
                                         chains.voxel ? 1.0f : 0.0f, post.cws, pass ? a.fallback_list : nullptr,
                                         pass ? l.hand_off_count() : nullptr, st, &launched, tab),
               RPL_RESULT_OPERATION_FAIL);
      c->launches += launched;
    }
    if (&l != &post && (r = scratch_leave(c, post, st)) != RPL_RESULT_OK) return r;
  }
  return scratch_leave(c, l, st);
}

// The cloud chain over the scans `a` of one chunk: its nodes, views, counts, nodes_total, n_scans and stride set (a
// push's chunk as its assembler left it, or last_push_scans); xyzi / point_counts point at the chunk's first slot;
// lidars: RPL_CLOUD_PER_STREAM's table at the chunk's first stream, lidar_scans slots per stream (else nullptr);
// chains: RPL_CLOUD_PER_STREAM_CHAIN's (the footprint table, chains_at(.., true), when footprints is set);
// footprints: RPL_CLOUD_PER_STREAM_FOOTPRINTS's table at the chunk's first stream (cloud_footprints_at; nullptr: no
// footprint pass).
// Flags 0: the shared-memory kernel with SOR / voxel grid fused, its arrays sized for at most kSmallPostMaxNodes nodes
// (a longer view goes to the general kernel, then to the post passes restricted to the hand-off list);
// RPL_CLOUD_NO_FUSED: the shared-memory kernel's window + xyz, then the post passes over every scan.
// RPL_CLOUD_PER_STREAM_CHAIN: the same per stream, by route -- the fused kernel for the fusable streams (when the call
// may fuse), the window-only kernel for the others; the post passes over every scan for the separate route, and
// restricted to the hand-off list for the fused route.  Each kernel and pass serves only its route's scans.
// With footprints, the footprint pass runs behind the scan kernels and before the post passes: without the chain flag
// the chunk runs as RPL_CLOUD_NO_FUSED, with it the footprint table routes every stream with a polygon separately.
rpl_result stream_cloud_chunk(rpl_ctx* c, Lane& l, rpl::ScanBatchArgs a, const rpl::LidarSettings* lidars,
                              const CloudChains& chains, uint32_t lidar_scans, const rpl_cloud_params* p, float* xyzi,
                              uint32_t* point_counts, cudaStream_t st, const rpl::ScanFootprint* footprints) {
  a.beam_counts = point_counts;
  a.fallback_list = l.fallback_list;
  a.is_new_protocol = p->is_new_protocol;
  a.xyzi = reinterpret_cast<float4*>(xyzi);
  a.trig = c->lane[0].cws.trig;
  a.angle = c->lane[0].cws.angle;
  a.range_min = p->range_min;
  a.range_max = p->range_max;
  a.intensity_min = p->intensity_min;
  a.lidar_scans = lidar_scans;
  if ((p->flags & RPL_CLOUD_PER_STREAM) != 0) a.lidars = lidars;  // each stream's is_new_protocol (the window's too)
  if ((p->flags & RPL_CLOUD_PER_STREAM_CHAIN) != 0)
    return stream_chains_chunk(c, l, a, chains, (p->flags & RPL_CLOUD_NO_FUSED) != 0, footprints, point_counts, st);
  const bool separate = (p->flags & RPL_CLOUD_NO_FUSED) != 0 || footprints;
  bool fused = false;
  rpl_result r = scratch_enter(c, l, st);
  if (r == RPL_RESULT_OK) r = enqueue_args(c, l, a, 0u, st, separate ? nullptr : p, &fused, true);
  if (r == RPL_RESULT_OK && footprints) r = footprint_clouds(c, a, footprints, rpl::ScanFootprint{}, point_counts, st);
  if (r != RPL_RESULT_OK) return r;
  if (p->sor_k > 0 || p->voxel_size > 0.0f) {
    // the post passes read lane l's fallback list and run on lane 0's cws: a lane-1 chunk takes lane 0's scratch too
    Lane& post = c->lane[0];
    if (&l != &post && (r = scratch_enter(c, post, st)) != RPL_RESULT_OK) return r;
    int launched = 0;
    RPL_CUDA(c, rpl::launch_cloud_post(a.xyzi, point_counts, a.n_scans, a.stride, p->sor_k, p->sor_alpha, p->voxel_size,
                                       post.cws, fused ? a.fallback_list : nullptr, fused ? l.hand_off_count() : nullptr,
                                       st, &launched),
             RPL_RESULT_OPERATION_FAIL);
    c->launches += launched;
    if (&l != &post && (r = scratch_leave(c, post, st)) != RPL_RESULT_OK) return r;
  }
  return scratch_leave(c, l, st);
}

// The device tables of the merge groups (rpl_capsule_stream_set_rescan_merges), carved from the session's mg_block:
// each stream's held row (kRescanMergeNone: in no group) and held grid, the grouped streams ascending, the members by
// group with each group's first member, the groups' max_age, the directory's choices, and the held rows
struct MergeTables {
  uint32_t* row;
  rpl::RescanHeld* held;
  uint32_t *streams, *members, *begin, *max_age, *pick;
  float* rows;
};
MergeTables merge_tables_layout(Carve& k, uint32_t n_streams, uint32_t n_grouped, uint32_t n_groups) {
  return MergeTables{k.take<uint32_t>(n_streams), k.take<rpl::RescanHeld>(n_streams), k.take<uint32_t>(n_grouped),
                     k.take<uint32_t>(n_grouped), k.take<uint32_t>(n_groups + 1), k.take<uint32_t>(n_groups),
                     k.take<uint32_t>(n_groups), k.take<float>((size_t)n_grouped * rpl::kRescanMaxBins)};
}
MergeTables merge_tables(const rpl_capsule_stream* cs) {
  Carve k{cs->mg_block};
  return merge_tables_layout(k, cs->n_streams, (uint32_t)cs->mg_streams_host.size(), cs->mg_groups);
}

// The re-grid of a LaserScan push's chunk (rpl_capsule_stream_push_rescan_msgs*), the session's tables at the chunk's
// first stream: the entries and their bins, the chunk's streams with a window and their windows, and for a merge push
// (rpl_capsule_stream_push_rescan_merge_msgs*) its grouped streams and their held grids
struct ChunkRescans {
  const rpl::RescanGrid* grid;  // nullptr: not a re-gridding push
  const uint32_t* bins;
  bool any;                     // an enabled entry in the chunk: rescan_kernel runs
  const uint32_t* streams;      // [n_win] session indices, from stream0 on
  uint32_t n_win, stream0;
  const rpl::RescanWindow* win;
  uint2* state;
  float* ring;
  const uint32_t* hold_streams;  // [n_hold] session indices
  uint32_t n_hold, seq;          // seq: the merge push's number
  const uint32_t* hold_row;
  rpl::RescanHeld* held;
  float* held_rows;
};

ChunkRescans rescan_chunk(const rpl_capsule_stream* cs, uint32_t s0, uint32_t ns, bool merge = false) {
  ChunkRescans r{};
  r.stream0 = s0;
  if (merge) {
    const std::vector<uint32_t>& gs = cs->mg_streams_host;
    const auto lo = std::lower_bound(gs.begin(), gs.end(), s0), hi = std::lower_bound(gs.begin(), gs.end(), s0 + ns);
    r.n_hold = (uint32_t)(hi - lo);
    if (r.n_hold) {
      const MergeTables t = merge_tables(cs);
      r.hold_streams = t.streams + (lo - gs.begin());
      r.seq = cs->mg_seq + 1;
      r.hold_row = t.row + s0;
      r.held = t.held + s0;
      r.held_rows = t.rows;
    }
  }
  r.grid = cs->rescan + s0;
  r.bins = cs->rescan_bins + s0;
  for (uint32_t s = s0; s < s0 + ns && !r.any; ++s) r.any = cs->rescan_host[s].enabled != 0;
  const std::vector<uint32_t>& ws = cs->win_streams_host;
  const auto lo = std::lower_bound(ws.begin(), ws.end(), s0), hi = std::lower_bound(ws.begin(), ws.end(), s0 + ns);
  r.n_win = (uint32_t)(hi - lo);
  if (r.n_win) {
    r.streams = cs->win_streams + (lo - ws.begin());
    r.win = cs->win + s0;
    r.state = cs->win_state + s0;
    r.ring = cs->win_ring;
  }
  return r;
}

// The projection of a LaserScan push's chunk (rpl_capsule_stream_push_scan_cloud_msgs*): its parameters (nullptr: none),
// the kept counts, and the clouds' messages and directory as a PointCloud2 push's (carry [2]; extent, total,
// extent_host and dir_order as ChunkMsgs'), every table at the chunk's first slot.  A re-gridding push
// (rescan.grid) takes the same members for its re-grid messages, and its own projection (the re-grid's points).
struct ChunkScanClouds {
  const rpl_scan_cloud_params* params;
  uint32_t* kept;
  uint8_t* out;
  unsigned long long capacity;
  unsigned long long *carry, *offsets, *extent, *total;
  uint32_t* sizes;
  unsigned long long* extent_host;
  cudaEvent_t dir_order;
  // RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS: the session's resolved headers and rows at the chunk's first stream
  const rpl::StreamMsgHeader* hdr;
  const float4* xf;
  ChunkRescans rescan;
};

// A message push's chunk (rpl_capsule_stream_push_{laserscan,cloud,scan_cloud}_msgs*): where its messages and tables
// go, every table at the chunk's first slot (stream).
struct ChunkMsgs {
  uint8_t* out;                      // LaserScan message i at out + place[i] - header - 32
  bool first, rebase;                // PushMsgDirArgs::first, rebase
  unsigned long long capacity;
  unsigned long long *carry, *offsets, *place, *extent, *total;  // PushMsgDirArgs (extent, total nullable)
  uint32_t* sizes;
  const rpl::StreamMsgHeader* hdr;
  long long clock_offset_ns;
  // a host push's: the directory's extent read back (pinned, then extent_ready), and the order of the chunks' directories
  // across the lanes (the previous chunk's directory recorded it)
  unsigned long long* extent_host;
  cudaEvent_t extent_ready, dir_order;
  // a PointCloud2 push's: the cloud chain's parameters and its clouds and point counts of the chunk's slots; message i
  // at out + offsets[i] - the base its writer is given (cloud_push_write)
  const rpl_cloud_params* cloud;
  float* xyzi;
  uint32_t* points;
  ChunkScanClouds proj;  // a LaserScan push's projected clouds
};

rpl::CloudTail cloud_tail();

// The projection of the LaserScan messages of the chunk of ns streams m describes, read where the push's scan kernels
// wrote them (m.out at m.place, m.sizes), with the header, stamps and timing laserscan_placed_kernel gave them: the
// count pass's arguments (the write pass adds the clouds' placement, scan_cloud_push_write)
rpl::ScanCloudArgs scan_cloud_push_args(const WireChunk& w, uint32_t ns, bool stamped, const rpl_scan_params* params,
                                        const ChunkMsgs& m, const uint32_t* beams, const float* inc) {
  rpl::ScanCloudArgs a{};
  scan_cloud_setup(a, *m.proj.params);
  a.m.hdr = m.hdr;
  if (stamped) {
    a.m.begin_us = w.slot_begin;
    a.m.end_us = w.slot_end;
  }
  a.m.clock_offset_ns = m.clock_offset_ns;
  a.m.counts = beams;
  a.m.angle_increment = inc;
  a.m.stride = w.max_nodes;
  a.m.max_scans = w.max_scans;
  a.m.mode_a = params->scan_processing ? 1u : 0u;
  a.m.lidars = w.lidars;
  a.m.n = ns * w.max_scans;
  a.kept = m.proj.kept;
  a.scan_msgs = m.out;
  a.place = m.place;
  a.scan_sizes = m.sizes;
  a.cloud_hdr = m.proj.hdr;
  a.xf = m.proj.xf;
  return a;
}

// the write pass of those clouds (a re-gridding push: of the re-grid messages), once their directory has placed them:
// message i at m.proj.out + offsets[i] - out_base
rpl_result scan_cloud_push_write(rpl_ctx* c, rpl::ScanCloudArgs a, const ChunkScanClouds& p, unsigned long long out_base,
                                 cudaStream_t st) {
  a.m.offsets = p.offsets;
  a.m.sizes = p.sizes;
  a.m.out = p.out;
  a.m.out_base = out_base;
  if (const ChunkRescans& q = p.rescan; q.grid) {
    rpl::RescanArgs ra{};
    ra.c = a;
    ra.grid = q.grid;
    if (q.any) {  // every message, as the replay re-grids it
      RPL_CUDA(c, rpl::launch_rescan(ra, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
      c->launches++;
    }
    if (q.n_win) {  // then the windows, over those grids (or their own, for a message that did not fit)
      rpl::RescanWindowArgs wa{};
      wa.r = ra;
      wa.streams = q.streams;
      wa.n = q.n_win;
      wa.stream0 = q.stream0;
      wa.win = q.win;
      wa.state = q.state;
      wa.ring = q.ring;
      RPL_CUDA(c, rpl::launch_rescan_window(wa, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
      c->launches++;
    }
    if (q.n_hold) {  // then the held grids, from the messages as published
      rpl::RescanHoldArgs ha{};
      ha.r = ra;
      ha.streams = q.hold_streams;
      ha.n = q.n_hold;
      ha.stream0 = q.stream0;
      ha.row = q.hold_row;
      ha.held = q.held;
      ha.rows = q.held_rows;
      ha.seq = q.seq;
      RPL_CUDA(c, rpl::launch_rescan_hold(ha, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
      c->launches++;
    }
    return RPL_RESULT_OK;
  }
  RPL_CUDA(c, rpl::launch_scan_cloud(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// A PointCloud2 push's messages of the chunk of ns streams m describes, once its directory has sized and placed them:
// pointcloud2_msgs_kernel writes message i at m.out + m.offsets[i] - out_base, stamped with the slot stamps of the
// stamped assembler (0 for an unstamped push), as msgs_write does for the last push's
rpl_result cloud_push_write(rpl_ctx* c, const WireChunk& w, uint32_t ns, bool stamped, const ChunkMsgs& m,
                            unsigned long long out_base, cudaStream_t st) {
  rpl::MsgWriteArgs a{};
  a.hdr = m.hdr;
  if (stamped) {
    a.begin_us = w.slot_begin;
    a.end_us = w.slot_end;
  }
  a.clock_offset_ns = m.clock_offset_ns;
  a.counts = m.points;
  a.xyzi = m.xyzi;
  a.stride = w.max_nodes;
  a.max_scans = w.max_scans;
  a.n = ns * w.max_scans;
  a.offsets = m.offsets;
  a.sizes = m.sizes;
  a.out = m.out;
  a.out_base = out_base;
  static const rpl::CloudTail tail = cloud_tail();
  RPL_CUDA(c, rpl::launch_pointcloud2_msgs(a, tail, w.max_nodes, st), RPL_RESULT_OPERATION_FAIL);
  c->launches += (a.n + 65534) / 65535;
  return RPL_RESULT_OK;
}

// (frame ->) decode -> assemble -> scan kernels for the ns streams of chunk w on `st`; capsules / counts / outputs / sp
// point at the chunk's first stream's (a byte session's capsules / counts: the raw bytes and byte counts).  A mixed
// byte session's chunk runs the first three for each answer type present in it, over that type's streams, and the scan
// kernels, which read the arenas whatever the type, once.
// m (a message push): the directory runs between the assembler and the scan kernels, which write into the placed
// messages instead of ranges / intens (null), and the header writer behind them.  A PointCloud2 push (m->cloud) runs
// the cloud chain over the chunk's fresh views instead of the scan kernels, then the directory, which sizes each
// message by its cloud, then (the device form; the host form's waits for the extent, push_host) the writer.  A LaserScan
// push with m->proj.params then projects the messages its header writer has finished: the count pass, the clouds'
// directory, and the write pass in the same way.
rpl_result capsule_stream_chunk(rpl_ctx* c, Lane& l, cudaStream_t st, const WireChunk& w, uint32_t ns,
                                const uint8_t* capsules, const uint32_t* counts, uint32_t sample_duration_us,
                                const rpl_scan_params* params, float* ranges, float* intens, uint32_t* beams,
                                float* inc, uint32_t* scans_per_stream, const StampPush* sp = nullptr,
                                const ChunkMsgs* m = nullptr) {
  rpl_result r = RPL_RESULT_OK;
  if (!w.list_begin) {
    r = decode_assemble(c, st, w, w.ans_type, ns, capsules, counts, sample_duration_us, scans_per_stream, sp, nullptr);
  } else {
    for (uint32_t t = 0; t < 6 && r == RPL_RESULT_OK; ++t) {
      const uint32_t b = w.list_begin[t], e = w.list_begin[t + 1];
      if (b == e) continue;
      const ListLaunch list{{w.lists + b, (uint32_t)w.framed_stride}, e - b};
      r = decode_assemble(c, st, w, RPL_ANS_MEASUREMENT + t, ns, capsules, counts, sample_duration_us,
                          scans_per_stream, sp, &list);
    }
  }
  if (r != RPL_RESULT_OK) return r;
  const LidarTable lt{w.lidars, w.max_scans, w.lidar_modes};
  const uint2* views = reinterpret_cast<const uint2*>(w.views);
  if (!m) {
    r = enqueue_scan(c, l, w.nodes, w.scan_len, ns * w.max_scans, w.max_nodes, params, nullptr, ranges, intens, beams,
                     inc, nullptr, nullptr, st, views, (unsigned long long)ns * w.stride_nodes, lt);
    if (r != RPL_RESULT_OK || !w.filters) return r;
    return filter_scans(c, w.filters, w.footprints, w.max_scans, ns * w.max_scans, ranges, intens, w.max_nodes,
                        nullptr, nullptr, beams, inc, st);
  }
  if (m->cloud) {  // the scans as last_push_scans will give them once the push is done
    rpl::ScanBatchArgs a{};
    a.nodes = reinterpret_cast<const uint2*>(w.nodes);
    a.views = views;
    a.counts = reinterpret_cast<const uint32_t*>(views);
    a.nodes_total = (unsigned long long)ns * w.stride_nodes;
    a.n_scans = ns * w.max_scans;
    a.stride = w.max_nodes;
    r = stream_cloud_chunk(c, l, a, w.lidars, w.clouds, w.max_scans, m->cloud, m->xyzi, m->points, st,
                           w.cloud_footprints);
    if (r != RPL_RESULT_OK) return r;
  }
  const rpl::MsgKind kind = m->cloud ? rpl::MsgKind::kPointCloud2 : rpl::MsgKind::kLaserScan;
  rpl::PushMsgDirArgs d{};
  d.views = views;
  d.scans_per_stream = scans_per_stream;
  d.hdr = m->hdr;
  d.n_slots = ns * w.max_scans;
  d.max_scans = w.max_scans;
  d.first = m->first ? 1u : 0u;
  d.rebase = m->rebase ? 1u : 0u;
  d.capacity = m->capacity;
  d.carry = m->carry;
  d.offsets = m->offsets;
  d.place = m->place;
  d.extent = m->extent;
  d.total = m->total;
  d.counts = m->points;
  d.sizes = m->cloud ? m->sizes : nullptr;
  if (m->cloud && (m->cloud->flags & RPL_CLOUD_PER_STREAM_CHAIN) != 0) d.clouds = w.clouds.at;
  // a directory behind the previous chunk's of its kind (a host push's order across the lanes), and its extent read back
  auto directory = [&](const rpl::PushMsgDirArgs& a, rpl::MsgKind k, cudaEvent_t order,
                       unsigned long long* extent_host) -> rpl_result {
    if (order) RPL_CUDA(c, cudaStreamWaitEvent(st, order, 0), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, rpl::launch_push_msg_dir(a, k, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
    if (order) RPL_CUDA(c, cudaEventRecord(order, st), RPL_RESULT_OPERATION_FAIL);
    if (extent_host) {
      RPL_CUDA(c, cudaMemcpyAsync(extent_host, a.extent, 3 * 8, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaEventRecord(m->extent_ready, st), RPL_RESULT_OPERATION_FAIL);
    }
    return RPL_RESULT_OK;
  };
  if (const rpl_result e = directory(d, kind, m->dir_order, m->extent_host); e != RPL_RESULT_OK) return e;
  if (m->cloud) return m->extent_host ? RPL_RESULT_OK : cloud_push_write(c, w, ns, sp != nullptr, *m, 0, st);
  r = enqueue_scan(c, l, w.nodes, w.scan_len, ns * w.max_scans, w.max_nodes, params, nullptr, nullptr, nullptr, beams,
                   inc, nullptr, nullptr, st, views, (unsigned long long)ns * w.stride_nodes, lt, m->out, m->place);
  if (r == RPL_RESULT_OK && w.filters)  // in place in the messages, before the header writer and the copies behind it
    r = filter_scans(c, w.filters, w.footprints, w.max_scans, ns * w.max_scans, nullptr, nullptr, 0, m->out, m->place,
                     beams, inc, st);
  if (r != RPL_RESULT_OK) return r;
  rpl::MsgWriteArgs a{};
  a.hdr = m->hdr;
  if (sp) {  // the slots' stamps, as the stamped assembler has just kept them
    a.begin_us = w.slot_begin;
    a.end_us = w.slot_end;
  }
  a.clock_offset_ns = m->clock_offset_ns;
  a.counts = beams;
  a.angle_increment = inc;
  a.max_scans = w.max_scans;
  a.mode_a = params->scan_processing ? 1u : 0u;
  a.n = ns * w.max_scans;
  a.out = m->out;
  a.lidars = w.lidars;
  RPL_CUDA(c, rpl::launch_laserscan_placed(a, m->place, m->sizes, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  if (!m->proj.params) return RPL_RESULT_OK;
  // the projection of the messages just finished: the kept counts, the clouds' directory, which sizes each message
  // exactly, then (the device form; the host form's waits for both extents, push_host) the write pass.  A re-gridding
  // push's directory sizes each re-grid message by its stream's entry: no count pass.
  const bool rescan = m->proj.rescan.grid != nullptr;
  const rpl::ScanCloudArgs sa = scan_cloud_push_args(w, ns, sp != nullptr, params, *m, beams, inc);
  if (!rescan) {
    RPL_CUDA(c, rpl::launch_scan_cloud_count(sa, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
  }
  d.capacity = m->proj.capacity;
  d.carry = m->proj.carry;
  d.offsets = m->proj.offsets;
  d.place = nullptr;
  d.extent = m->proj.extent;
  d.total = m->proj.total;
  d.counts = m->proj.kept;
  d.sizes = m->proj.sizes;
  d.scan_sizes = m->sizes;
  if (sa.transform) d.hdr = m->proj.hdr;  // the target frames' headers size the messages
  d.tail_bytes = sa.transform ? sa.tail_xf.bytes : sa.tail.bytes;
  d.point_step = sa.point_step;
  if (rescan) d.counts = m->proj.rescan.bins;
  r = directory(d, rescan ? rpl::MsgKind::kRescan : rpl::MsgKind::kScanCloud, m->proj.dir_order, m->proj.extent_host);
  if (r != RPL_RESULT_OK || m->extent_host) return r;
  return scan_cloud_push_write(c, sa, m->proj, 0, st);
}

struct HostMsgs;

// A host call's wire input and LaserScan outputs: host arrays of all its streams (the chain's, a session's host push)
struct HostWire {
  const uint8_t* capsules;  // [n_streams][in_stream bytes]
  const uint32_t* counts;
  size_t in_stream;
  uint32_t sample_duration_us, max_nodes, max_scans;
  const rpl_scan_params* params;
  float *ranges, *intensities, *angle_increment;  // angle_increment nullable
  uint32_t *beam_counts, *scans_per_stream;
  const StampPush* sp;  // a stamped push: receive times in, scan stamps out
  size_t rx_stream;     // receive times per stream of a stamped push
  const HostMsgs* msgs;  // a message push: its messages instead of the LaserScan rows (ranges etc. unused)
};

// A host message push's outputs (host arrays of every slot) and the session's device tables of its chunks
struct HostMsgs {
  uint8_t* msgs;
  unsigned long long capacity;
  uint64_t* offsets;
  uint32_t* sizes;
  uint64_t* total;
  size_t chunk_bytes;  // staging for one chunk's messages: the bound of its slots at max_nodes
  long long clock_offset_ns;
  const rpl::StreamMsgHeader* hdr;  // the session's, [n_streams]
  unsigned long long *carry, *place;
  unsigned long long* extent_host;  // [kLanes][3] pinned, and extent_ready[kLanes]: each lane's chunk's
  const cudaEvent_t* extent_ready;
  cudaEvent_t dir_order;
  const rpl_cloud_params* cloud;    // a PointCloud2 push
  // a LaserScan push that also projects its scans: the projection's parameters, the clouds' outputs, the staging for
  // one chunk's clouds (their bound at max_nodes), the session's cloud carry and kept counts, each lane's cloud extent
  // (pinned [kLanes][3], ready with extent_ready) and the order of the cloud directories
  const rpl_scan_cloud_params* proj;
  const rpl_msgs_out* clouds;
  size_t proj_chunk_bytes;
  unsigned long long *proj_carry, *proj_extent_host;
  uint32_t* kept;
  cudaEvent_t proj_dir_order;
  const rpl::StreamMsgHeader* proj_hdr;  // RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS: the session's resolved headers, rows
  const float4* proj_xf;
  // a re-gridding push: its session (rescan_chunk), whose re-grid messages take the projection's members above; merge:
  // a merge push, which holds the grouped streams' grids
  const rpl_capsule_stream* rescan;
  bool merge;
};

// Runs a host call's n_streams streams through capsule_stream_chunk, `chunk` streams at a time round-robin over the
// lanes: H2D of a chunk's input (and receive times), its kernels, D2H of its LaserScans (and stamps).  A message push
// (h.msgs) stages the chunk's messages instead: once its directory's extent is read back (the chunk's scan kernels run
// meanwhile), the stretch of the packed buffer the chunk fills is copied to msgs, with the chunk's tables.  A
// PointCloud2 push's directory follows the chunk's cloud kernels, so the host reads a chunk's extent only once the next
// chunk is queued on the other lane (finish_cloud), then queues the writer, which packs the chunk's messages from the
// stretch's first offset on, and the copies.  A projecting push (hm->proj) does the same for its clouds, whose
// directory follows the chunk's scan kernels: both extents are read once the next chunk is queued, then the clouds'
// write pass and both stretches and tables are queued.  A lane's staging block holds one chunk's input and outputs,
// then whatever chunk_at(k, s0) carves off k for the device state of the chunk from stream s0, which it returns (the
// chain's lives there; a session's in its arenas).
template <class ChunkAt>
rpl_result push_host(rpl_ctx* c, const HostWire& h, uint32_t n_streams, uint32_t chunk, ChunkAt chunk_at) {
  const size_t NS = (size_t)chunk * h.max_scans, row = (size_t)h.max_scans * h.max_nodes;
  using u64 = unsigned long long;
  const HostMsgs* hm = h.msgs;
  const size_t rows = hm ? 0 : NS * h.max_nodes;
  struct Regions {
    uint8_t* in;
    uint32_t* counts;
    u64* rx;
    float *ranges, *intens, *inc;
    uint32_t *beams, *sps;
    u64* ts;
    uint8_t* msgs;  // a message push's: the chunk's messages, offsets, sizes and extent
    u64* offs;
    uint32_t* sizes;
    u64* extent;
    float* xyzi;  // a PointCloud2 push's: the chunk's clouds and point counts
    uint32_t* points;
    uint8_t* pmsgs;  // a projecting push's: the chunk's projected clouds, their offsets, sizes and extent
    u64* poffs;
    uint32_t* psizes;
    u64* pextent;
    WireChunk w;
  };
  const bool cloud = hm && hm->cloud, proj = hm && hm->proj;
  auto layout = [&](Carve& k, uint32_t s0) {
    return Regions{k.take<uint8_t>(chunk * h.in_stream), k.take<uint32_t>(chunk),
                   k.take<u64>(h.sp ? chunk * h.rx_stream : 0), k.take<float>(rows), k.take<float>(rows),
                   k.take<float>(NS), k.take<uint32_t>(NS), k.take<uint32_t>(chunk), k.take<u64>(h.sp ? NS : 0),
                   k.take<uint8_t>(hm ? hm->chunk_bytes : 0), k.take<u64>(hm ? NS : 0), k.take<uint32_t>(hm ? NS : 0),
                   k.take<u64>(hm ? 3 : 0), k.take<float>(cloud ? NS * h.max_nodes * 4 : 0),
                   k.take<uint32_t>(cloud ? NS : 0), k.take<uint8_t>(proj ? hm->proj_chunk_bytes : 0),
                   k.take<u64>(proj ? NS : 0), k.take<uint32_t>(proj ? NS : 0), k.take<u64>(proj ? 3 : 0),
                   chunk_at(k, s0)};
  };
  if (const rpl_result r = grow_stage(c, kLanes, [&](Carve& k) { layout(k, 0); }); r != RPL_RESULT_OK) return r;
  const cudaMemcpyKind h2d = cudaMemcpyHostToDevice, d2h = cudaMemcpyDeviceToHost;
  // a PointCloud2 or projecting push's chunk whose kernels are queued and whose writer and copies are not
  struct Queued {
    Lane* l = nullptr;
    uint32_t s0, ns;
    Regions d;
    ChunkMsgs m;
  } queued;
  auto finish_cloud = [&]() -> rpl_result {
    if (!queued.l) return RPL_RESULT_OK;
    const Queued q = queued;
    queued.l = nullptr;
    const int li = (int)(q.l - c->lane);
    const size_t so = (size_t)q.s0 * h.max_scans, nsc = (size_t)q.ns * h.max_scans;
    const bool last = q.s0 + q.ns == n_streams;
    cudaStream_t st = q.l->stream;
    RPL_CUDA(c, cudaEventSynchronize(hm->extent_ready[li]), RPL_RESULT_OPERATION_FAIL);
    const u64 lo = q.m.extent_host[0], hi = q.m.extent_host[1];
    if (last) *hm->total = q.m.extent_host[2];
    if (cloud)
      if (const rpl_result r = cloud_push_write(c, q.d.w, q.ns, h.sp != nullptr, q.m, lo, st); r != RPL_RESULT_OK)
        return r;
    if (proj) {  // the clouds' stretch [first offset, end of the last that fits), written from its first offset on
      const u64 plo = q.m.proj.extent_host[0], phi = q.m.proj.extent_host[1];
      if (last) *hm->clouds->total_bytes = q.m.proj.extent_host[2];
      const rpl::ScanCloudArgs a = scan_cloud_push_args(q.d.w, q.ns, h.sp != nullptr, h.params, q.m, q.d.beams, q.d.inc);
      if (const rpl_result r = scan_cloud_push_write(c, a, q.m.proj, plo, st); r != RPL_RESULT_OK) return r;
      if (phi > plo)
        RPL_CUDA(c, cudaMemcpyAsync(hm->clouds->msgs + plo, q.d.pmsgs, phi - plo, d2h, st), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(hm->clouds->msg_offsets + so, q.d.poffs, nsc * 8, d2h, st), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(hm->clouds->msg_sizes + so, q.d.psizes, nsc * 4, d2h, st), RPL_RESULT_OPERATION_FAIL);
    }
    if (hi > lo) RPL_CUDA(c, cudaMemcpyAsync(hm->msgs + lo, q.d.msgs, hi - lo, d2h, st), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(hm->offsets + so, q.d.offs, nsc * 8, d2h, st), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(hm->sizes + so, q.d.sizes, nsc * 4, d2h, st), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(h.scans_per_stream + q.s0, q.d.sps, (size_t)q.ns * 4, d2h, st),
             RPL_RESULT_OPERATION_FAIL);
    return RPL_RESULT_OK;
  };
  auto run_chunk = [&](Lane& l, uint32_t s0, uint32_t ns) -> rpl_result {
    Carve k{l.stage};
    const Regions d = layout(k, s0);
    const size_t so = (size_t)s0 * h.max_scans, nsc = (size_t)ns * h.max_scans;
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);  // the lane's previous chunk has left
    RPL_CUDA(c, cudaMemcpyAsync(d.in, h.capsules + s0 * h.in_stream, ns * h.in_stream, h2d, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(d.counts, h.counts + s0, (size_t)ns * 4, h2d, l.stream), RPL_RESULT_OPERATION_FAIL);
    StampPush sp{};
    if (h.sp) {
      sp = *h.sp;
      sp.rx = d.rx;
      sp.scan_ts = d.ts;
      RPL_CUDA(c, cudaMemcpyAsync(d.rx, h.sp->rx + s0 * h.rx_stream, ns * h.rx_stream * 8, h2d, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    }
    ChunkMsgs m{};
    if (hm) {
      m.out = d.msgs;
      m.first = s0 == 0;
      m.rebase = true;
      m.capacity = hm->capacity;
      m.carry = hm->carry;
      m.offsets = d.offs;
      m.place = hm->place + so;
      m.extent = d.extent;
      m.sizes = d.sizes;
      m.hdr = hm->hdr + s0;
      m.clock_offset_ns = hm->clock_offset_ns;
      const int li = (int)(&l - c->lane);
      m.extent_host = hm->extent_host + 3 * li;
      m.extent_ready = hm->extent_ready[li];
      m.dir_order = hm->dir_order;
      m.cloud = hm->cloud;
      m.xyzi = d.xyzi;
      m.points = d.points;
      if (proj)
        m.proj = ChunkScanClouds{hm->proj, hm->kept + so, d.pmsgs, hm->clouds->capacity, hm->proj_carry, d.poffs,
                                 d.pextent, nullptr, d.psizes, hm->proj_extent_host + 3 * li, hm->proj_dir_order,
                                 hm->proj_hdr ? hm->proj_hdr + s0 : nullptr, hm->proj_xf ? hm->proj_xf + 3 * s0 : nullptr};
      if (proj && hm->rescan) m.proj.rescan = rescan_chunk(hm->rescan, s0, ns, hm->merge);
    }
    const rpl_result r = capsule_stream_chunk(c, l, l.stream, d.w, ns, d.in, d.counts, h.sample_duration_us, h.params,
                                              d.ranges, d.intens, d.beams, d.inc, d.sps, h.sp ? &sp : nullptr,
                                              hm ? &m : nullptr);
    if (r != RPL_RESULT_OK) return r;
    if (cloud || proj) {  // this chunk runs while the host waits for the previous one's extent
      const rpl_result f = finish_cloud();
      queued = Queued{&l, s0, ns, d, m};
      return f;
    }
    if (hm) {
      // the chunk's stretch [first offset, end of its last message that fits): known once its directory has run
      RPL_CUDA(c, cudaEventSynchronize(m.extent_ready), RPL_RESULT_OPERATION_FAIL);
      const u64 lo = m.extent_host[0], hi = m.extent_host[1];
      if (s0 + ns == n_streams) *hm->total = m.extent_host[2];
      if (hi > lo)
        RPL_CUDA(c, cudaMemcpyAsync(hm->msgs + lo, d.msgs, hi - lo, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(hm->offsets + so, d.offs, nsc * 8, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(hm->sizes + so, d.sizes, nsc * 4, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
      RPL_CUDA(c, cudaMemcpyAsync(h.scans_per_stream + s0, d.sps, (size_t)ns * 4, d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
      return RPL_RESULT_OK;
    }
    if (h.sp)
      RPL_CUDA(c, cudaMemcpyAsync(h.sp->scan_ts + so, d.ts, nsc * 8, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(h.ranges + so * h.max_nodes, d.ranges, ns * row * 4, d2h, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(h.intensities + so * h.max_nodes, d.intens, ns * row * 4, d2h, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(h.beam_counts + so, d.beams, nsc * 4, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
    if (h.angle_increment)
      RPL_CUDA(c, cudaMemcpyAsync(h.angle_increment + so, d.inc, nsc * 4, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(h.scans_per_stream + s0, d.sps, (size_t)ns * 4, d2h, l.stream),
             RPL_RESULT_OPERATION_FAIL);
    return RPL_RESULT_OK;
  };
  rpl_result r = run_chunks(c, n_streams, chunk, run_chunk);
  if (r == RPL_RESULT_OK && queued.l) {  // the last chunk of a PointCloud2 or projecting push
    r = finish_cloud();
    const std::string why = c->err;
    const rpl_result s = rpl_ctx_synchronize(c);
    if (r == RPL_RESULT_OK) return s;
    c->err = why;
  }
  return r;
}

// The tables of a nodes call (rpl_capsule_stream_nodes*), the session's own: every slot's place for the kernels, the
// per-stream ascend flags, and the host form's directory, which the device form writes into the caller's arrays.
struct NodeWork {
  unsigned long long *place, *offsets, *total;
  uint32_t *counts, *status;
  uint8_t* ascend;
};
NodeWork node_work_layout(const rpl_capsule_stream* cs, Carve& k) {
  const size_t NS = (size_t)cs->n_streams * cs->max_scans;
  return NodeWork{k.take<unsigned long long>(NS), k.take<unsigned long long>(NS), k.take<unsigned long long>(1),
                  k.take<uint32_t>(NS), k.take<uint32_t>(NS), k.take<uint8_t>(cs->n_streams)};
}
size_t node_work_bytes(const rpl_capsule_stream* cs) {
  Carve k;
  node_work_layout(cs, k);
  return k.bytes;
}

// a call with RPL_FLAG_PER_STREAM / RPL_CLOUD_PER_STREAM needs the table
bool lidars_ok(rpl_capsule_stream* cs) {
  if (!cs->lidars_host.empty()) return true;
  cs->c->err = "per-stream settings requested before rpl_*_stream_set_lidars set every stream";
  return false;
}

// a call with RPL_FLAG_PER_STREAM_FILTERS needs the table
bool filters_ok(rpl_capsule_stream* cs) {
  if (!cs->filters_host.empty()) return true;
  cs->c->err = "per-stream scan filters requested before rpl_capsule_stream_set_scan_filters set every stream";
  return false;
}

// the table of a session call: the stream s0's entry on, when per_stream
LidarTable lidar_table(const rpl_capsule_stream* cs, bool per_stream, uint32_t s0) {
  if (!per_stream) return LidarTable{};
  return LidarTable{cs->lidars + s0, cs->max_scans, cs->lidar_modes};
}

// the table's entry of stream s0, nullptr before the first set_lidars
const rpl::LidarSettings* lidars_at(const rpl_capsule_stream* cs, uint32_t s0) {
  return cs->lidars ? cs->lidars + s0 : nullptr;
}

// a capsule answer type's decoder runs in the session's pushes (a mixed session's: any stream's)
bool decodes_capsules(const rpl_capsule_stream* cs) {
  if (cs->types.empty()) return cs->ans_type != RPL_ANS_MEASUREMENT;
  return std::any_of(cs->types.begin(), cs->types.end(), [](uint32_t t) { return t != RPL_ANS_MEASUREMENT; });
}

// msgs: a message push, which has no LaserScan rows
bool capsule_stream_args_ok(rpl_capsule_stream* cs, const uint8_t* capsules, const uint32_t* capsule_counts,
                            uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                            float* intensities, uint32_t* beam_counts, uint32_t* scans_per_stream, bool msgs = false) {
  rpl_ctx* c = cs->c;
  if (!capsules || !capsule_counts || !params || (!msgs && (!ranges || !intensities || !beam_counts)) ||
      !scans_per_stream) {
    c->err = "null capsules, counts, params or output buffer";
    return false;
  }
  if ((params->flags & RPL_FLAG_PER_STREAM_FILTERS) != 0 && !filters_ok(cs)) return false;
  if ((params->flags & RPL_FLAG_PER_STREAM) != 0) {  // every stream's sample duration comes from the table
    if (!lidars_ok(cs)) return false;
  } else if (decodes_capsules(cs) && !sample_duration_ok(c, sample_duration_us)) {
    // (the standard decoder takes no sample duration: it tests no jump between capsules)
    return false;
  }
  // the alignment rule of rpl_decode_capsules_batch_dev: only dense capsules are read in 4-byte words (a byte session's
  // bytes have any alignment: its decoder reads the session's own capsule slots)
  if (cs->ans_type == 0x85 && !cs->bytes && (reinterpret_cast<uintptr_t>(capsules) & 3u) != 0) {
    c->err = "capsule buffer must be 4-byte aligned";
    return false;
  }
  return true;
}

// a stream's message settings: XCDR1 encapsulation {0x00, 0x01, 0x00, 0x00}, a zero stamp, frame_id as a string
// (uint32 length with the NUL, the bytes, the NUL), zero padding to 4
rpl::StreamMsgHeader msg_header(const char* frame_id, size_t len, float range_max) {
  rpl::StreamMsgHeader h{};
  uint8_t* b = reinterpret_cast<uint8_t*>(h.w);
  b[1] = 0x01;
  const uint32_t n = (uint32_t)len + 1;
  std::memcpy(b + 12, &n, 4);
  std::memcpy(b + 16, frame_id, len);
  h.bytes = 4 + ((12 + (uint32_t)len + 1 + 3) & ~3u);
  h.range_max = range_max;
  return h;
}

// a mixed byte session's answer types: each chunking's lists and directory, built from t and uploaded (synchronously:
// no device call of the session may be in flight)
rpl_result set_types(rpl_capsule_stream* cs, std::vector<uint32_t> t) {
  rpl_ctx* c = cs->c;
  std::vector<uint32_t> lists[2];
  std::vector<uint32_t> begin[2];
  for (int k = 0; k < 2; ++k) {
    const uint32_t chunk = k ? cs->chunk_dev : cs->chunk_host;
    lists[k].reserve(cs->n_streams);
    for (uint32_t s0 = 0; s0 < cs->n_streams; s0 += chunk) {
      const uint32_t ns = std::min(chunk, cs->n_streams - s0);
      for (uint32_t y = 0; y < 6; ++y) {
        begin[k].push_back((uint32_t)lists[k].size() - s0);
        for (uint32_t i = 0; i < ns; ++i)
          if (t[s0 + i] == RPL_ANS_MEASUREMENT + y) lists[k].push_back(i);
      }
      begin[k].push_back(ns);
    }
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  cudaStream_t st = c->lane[0].stream;
  for (int k = 0; k < 2; ++k)
    RPL_CUDA(c, cudaMemcpyAsync(cs->lists[k], lists[k].data(), lists[k].size() * 4, cudaMemcpyHostToDevice, st),
             RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  for (int k = 0; k < 2; ++k) cs->list_begin[k] = std::move(begin[k]);
  cs->types = std::move(t);
  return RPL_RESULT_OK;
}

// The per-stream regions of a session of answer type ans_type whose pushes take at most stride_in framed capsules, or
// with `bytes` at most stride_in bytes of the serial stream: capsule slots and the nodes one push may complete
struct StreamSizes {
  unsigned long long stride_capsules, new_nodes;
};
StreamSizes stream_sizes(uint32_t ans_type, bool bytes, uint32_t stride_in) {
  const bool normal = ans_type == RPL_ANS_MEASUREMENT, framing = bytes && !normal;
  const uint32_t cap_bytes = normal ? 1u : rpl_capsule_bytes(ans_type);
  // a byte push completes at most `frames` frames with the up to cap_bytes - 1 bytes held before it, each behind at most
  // one all-zero capsule (none for HQ, whose skipped bytes are no loss)
  const unsigned long long frames = framing ? ((unsigned long long)stride_in + cap_bytes - 1) / cap_bytes : stride_in;
  const unsigned long long stride_capsules = framing ? (ans_type == 0x83 ? frames : 2 * frames) : stride_in;
  // 0x81: a push of n bytes completes up to (n + 4) / 5 records with the up to 4 bytes held before it; rounded up to
  // even, as every capsule format's node count is, so that every region stays 16-byte aligned
  const unsigned long long new_nodes = normal ? ((stride_capsules + 4) / 5 + 1) & ~1ull
                                              : (unsigned long long)rpl_capsule_nodes(ans_type) * frames;
  return StreamSizes{stride_capsules, new_nodes};
}

// a session of answer type ans_type (the caller has checked it) whose pushes take, per stream, at most stride_in framed
// capsules, or with `bytes` at most stride_in bytes of the serial stream (a capsule answer type's are framed first).
// types (a mixed byte session, ans_type 0 and `bytes`): each stream's answer type, every region sized for the largest
// any of the six types needs
rpl_result stream_create(rpl_ctx* c, uint32_t ans_type, bool bytes, uint32_t n_streams, uint32_t stride_in,
                         uint32_t max_nodes, uint32_t max_scans, rpl_capsule_stream** out,
                         const uint32_t* types = nullptr) {
  const bool normal = ans_type == RPL_ANS_MEASUREMENT, framing = bytes && !normal;
  const uint32_t cap_bytes = normal || types ? 1u : rpl_capsule_bytes(ans_type);
  StreamSizes z{0, 0};
  unsigned long long framed_stride = 0;
  if (!types) {
    z = stream_sizes(ans_type, bytes, stride_in);
    framed_stride = framing ? z.stride_capsules * cap_bytes : 0;
  } else {
    for (uint32_t t = RPL_ANS_MEASUREMENT; t <= 0x86u; ++t) {
      const StreamSizes y = stream_sizes(t, true, stride_in);
      z.new_nodes = std::max(z.new_nodes, y.new_nodes);
      if (t == RPL_ANS_MEASUREMENT) continue;  // its decoder reads the pushed bytes: no capsule slots
      z.stride_capsules = std::max(z.stride_capsules, y.stride_capsules);
      framed_stride = std::max(framed_stride, y.stride_capsules * rpl_capsule_bytes(t));
    }
    framed_stride = (framed_stride + 15) & ~15ull;  // every stream's capsules 16-byte aligned
  }
  if (types && framed_stride > 0xFFFFFFFFull) {  // StreamList::capsule_stride
    c->err = "stride_bytes too large: a stream's framed capsules must stay below 2^32 bytes";
    return RPL_RESULT_INVALID_DATA;
  }
  const uint32_t stride_capsules = (uint32_t)z.stride_capsules;
  if (n_streams == 0 || stride_capsules == 0 || max_scans == 0 || max_nodes == 0 || max_nodes > rpl::kSmallMaxNodes ||
      (max_nodes & 1u)) {
    c->err = bytes ? "need n_streams > 0, stride_bytes > 0, max_scans > 0 and an even max_nodes in [2, 8192]"
                   : "need n_streams > 0, stride_capsules > 0, max_scans > 0 and an even max_nodes in [2, 8192]";
    return RPL_RESULT_INVALID_DATA;
  }
  if (max_scans > c->max_scans) {
    c->err = "the context's max_scans is smaller than max_scans of one stream";
    return RPL_RESULT_INVALID_DATA;
  }
  const unsigned long long new_nodes = z.new_nodes;
  const unsigned long long stride_nodes = (unsigned long long)max_nodes + new_nodes;
  if (stride_nodes * n_streams > 0xFFFFFFFFull) {
    c->err = types ? "n_streams * (max_nodes + 96 * ceil(stride_bytes / 132)) must stay below 2^32 (32-bit scan views)"
           : normal ? "n_streams * (max_nodes + (stride_bytes + 4) / 5 rounded up to even) must stay below 2^32 "
                      "(32-bit scan views)"
                    : framing ? "n_streams * (max_nodes + nodes per capsule * ceil(stride_bytes / capsule bytes)) must "
                                "stay below 2^32 (32-bit scan views)"
                              : "n_streams * (max_nodes + nodes per capsule * stride_capsules) must stay below 2^32 "
                                "(32-bit scan views)";
    return RPL_RESULT_INVALID_DATA;
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  rpl_capsule_stream* cs = new (std::nothrow) rpl_capsule_stream();
  if (!cs) return RPL_RESULT_INSUFFICIENT_MEMORY;
  cs->c = c;
  cs->ans_type = ans_type;
  cs->cap_bytes = cap_bytes;
  cs->framed_stride = (size_t)framed_stride;
  cs->n_streams = n_streams;
  cs->stride_capsules = stride_capsules;
  cs->max_nodes = max_nodes;
  cs->max_scans = max_scans;
  cs->stride_nodes = (uint32_t)stride_nodes;  // even: every region starts 16-byte aligned
  cs->starts_stride = 2 * max_scans + 64;     // scan starts per stream the decoder may list (as in the chain)
  cs->chunk_dev = std::min(n_streams, c->max_scans / max_scans);
  cs->bytes = bytes;
  cs->stride_in = stride_in;
  cs->in_stream = bytes ? (size_t)stride_in : (size_t)stride_in * cap_bytes;
  // host pushes: about 16 MiB of capsules (a byte session: bytes) per chunk, whole streams (as in the chain)
  cs->chunk_host = std::min<uint32_t>(cs->chunk_dev, (uint32_t)std::max<size_t>(1, ((size_t)16 << 20) / cs->in_stream));
  const size_t n = n_streams, ncap = n * stride_capsules;
  const rpl_result oom = RPL_RESULT_INSUFFICIENT_MEMORY;
  auto fail = [&](rpl_result r) {
    rpl_capsule_stream_destroy(cs);
    return r;
  };
  for (int p = 0; p < 2; ++p)
    if (!cuda_ok(c, dev_alloc(&cs->arena[p], n * cs->stride_nodes), "cudaMalloc") ||
        !cuda_ok(c, dev_alloc(&cs->carry_len[p], n), "cudaMalloc") ||
        !cuda_ok(c, cudaMemset(cs->carry_len[p], 0, n * 4), "cudaMemset") ||
        !cuda_ok(c, dev_alloc(&cs->open_ts[p], n), "cudaMalloc") ||
        !cuda_ok(c, cudaMemset(cs->open_ts[p], 0, n * 8), "cudaMemset"))
      return fail(oom);
  if (!cuda_ok(c, dev_alloc(&cs->held_rx, n), "cudaMalloc") ||
      !cuda_ok(c, cudaMemset(cs->held_rx, 0, n * 8), "cudaMemset"))
    return fail(oom);
  if ((normal || types) && !cuda_ok(c, dev_alloc(&cs->scan_ends, n * (size_t)new_nodes), "cudaMalloc")) return fail(oom);
  if ((ans_type == 0x85 || types) && (!cuda_ok(c, dev_alloc(&cs->starts, n * cs->starts_stride), "cudaMalloc") ||
                           !cuda_ok(c, dev_alloc(&cs->start_counts, n), "cudaMalloc")))
    return fail(oom);
  if (!normal && (!cuda_ok(c, dev_alloc(&cs->status, ncap), "cudaMalloc") ||
                  !cuda_ok(c, dev_alloc(&cs->offsets, ncap), "cudaMalloc")))
    return fail(oom);
  if (framing && (!cuda_ok(c, dev_alloc(&cs->framer, n * rpl::kFramerWords), "cudaMalloc") ||
                  !cuda_ok(c, cudaMemset(cs->framer, 0, n * rpl::kFramerWords * 4), "cudaMemset") ||
                  !cuda_ok(c, dev_alloc(&cs->framed, n * framed_stride), "cudaMalloc") ||
                  !cuda_ok(c, dev_alloc(&cs->framed_counts, n), "cudaMalloc") ||
                  !cuda_ok(c, dev_alloc(&cs->framed_rx, ncap), "cudaMalloc")))
    return fail(oom);
  if (!cuda_ok(c, dev_alloc(&cs->held, n * rpl::kHeldWords), "cudaMalloc") ||
      !cuda_ok(c, cudaMemset(cs->held, 0, n * rpl::kHeldWords * 4), "cudaMemset") ||
      !cuda_ok(c, dev_alloc(&cs->node_counts, n), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->scan_len, n * max_scans), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->views, n * max_scans), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->slot_begin, n * max_scans), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->slot_end, n * max_scans), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->msg_hdr, n), "cudaMalloc") ||
      !cuda_ok(c, dev_alloc(&cs->counters, n), "cudaMalloc") ||
      !cuda_ok(c, cudaMemset(cs->counters, 0, n * sizeof(rpl::StreamCounters)), "cudaMemset") ||
      !cuda_ok(c, dev_alloc(&cs->node_work, node_work_bytes(cs)), "cudaMalloc"))
    return fail(oom);
  // the reference's defaults: frame_id "laser_frame" (rplidar_node.cpp:80), range_max 12 m (rplidar_node.hpp:328)
  cs->msg_hdr_host.assign(n, msg_header("laser_frame", 11, 12.0f));
  if (!cuda_ok(c, cudaMemcpy(cs->msg_hdr, cs->msg_hdr_host.data(), n * sizeof(rpl::StreamMsgHeader),
                             cudaMemcpyHostToDevice), "cudaMemcpy") ||
      !cuda_ok(c, cudaEventCreateWithFlags(&cs->done, cudaEventDisableTiming), "cudaEventCreate") ||
      !cuda_ok(c, cudaDeviceSynchronize(), "cudaDeviceSynchronize"))  // the zeroed state is in place before any push
    return fail(oom);
  if (types) {
    for (int k = 0; k < 2; ++k)
      if (!cuda_ok(c, dev_alloc(&cs->lists[k], n), "cudaMalloc")) return fail(oom);
    if (const rpl_result r = set_types(cs, std::vector<uint32_t>(types, types + n_streams)); r != RPL_RESULT_OK)
      return fail(r);
  }
  *out = cs;
  return RPL_RESULT_OK;
}

// the stamped pushes' own arguments (chunk_bytes: the byte pushes', 1 for a framed push) into *sp; with
// RPL_FLAG_PER_STREAM the table's timing serves and `timing` may be null
bool stamp_args_ok(rpl_capsule_stream* cs, const rpl_scan_params* params, const rpl_timing* timing, const uint64_t* rx,
                   uint32_t chunk_bytes, uint64_t* scan_begin_ts_us, StampPush* sp) {
  if (!cs) return false;
  rpl_ctx* c = cs->c;
  const bool per_stream = params && (params->flags & RPL_FLAG_PER_STREAM) != 0;
  if ((!timing && !per_stream) || !rx || !scan_begin_ts_us) {
    c->err = "null timing, receive times or scan_begin_ts_us";
    return false;
  }
  if (chunk_bytes == 0) {
    c->err = "chunk_bytes must be > 0";
    return false;
  }
  if (misaligned8(rx) || misaligned8(scan_begin_ts_us)) {
    c->err = "timestamp buffers must be 8-byte aligned";
    return false;
  }
  if (timing && !per_stream)
    sp->timing = rpl::TimingDesc{timing->sample_duration_us, timing->native_baudrate, timing->linkage_delay_us,
                                 timing->native_interface_type};
  sp->rx = reinterpret_cast<const unsigned long long*>(rx);
  sp->chunk_bytes = chunk_bytes;
  sp->stride_chunks = (uint32_t)(((unsigned long long)cs->stride_in + chunk_bytes - 1) / chunk_bytes);
  sp->scan_ts = reinterpret_cast<unsigned long long*>(scan_begin_ts_us);
  return true;
}

// a byte push on a framed session or a framed push on a byte session
bool push_kind_ok(rpl_capsule_stream* cs, bool bytes) {
  if (cs->bytes == bytes) return true;
  cs->c->err = bytes ? "a byte push needs a session made by rpl_capsule_stream_create_bytes"
                     : "a session made by rpl_capsule_stream_create_bytes takes byte pushes (rpl_capsule_stream_push_bytes*)";
  return false;
}

// The session's device tables of a message push, every slot's: the carry of the directories (a PointCloud2 push's: the
// running offset and the end of the last message), each slot's place, the scan kernels' beam counts and angle
// increments, and the stamped assembler's scan stamps
struct PushMsgWork {
  unsigned long long *carry, *place;
  uint32_t* beams;
  float* inc;
  unsigned long long* ts;
};
PushMsgWork push_msg_work_layout(const rpl_capsule_stream* cs, Carve& k) {
  const size_t NS = (size_t)cs->n_streams * cs->max_scans;
  return PushMsgWork{k.take<unsigned long long>(2), k.take<unsigned long long>(NS), k.take<uint32_t>(NS),
                     k.take<float>(NS), k.take<unsigned long long>(NS)};
}

// The session's device tables of a projecting push: the clouds' directory carry (the running offset and the end of
// the last message) and every slot's kept count
struct ScanCloudWork {
  unsigned long long* carry;
  uint32_t* kept;
};
ScanCloudWork scan_cloud_work_layout(const rpl_capsule_stream* cs, Carve& k) {
  return ScanCloudWork{k.take<unsigned long long>(2), k.take<uint32_t>((size_t)cs->n_streams * cs->max_scans)};
}

// a message push's outputs (host or device arrays of every slot, as the push's)
struct PushMsgs {
  uint8_t* msgs;
  unsigned long long capacity;
  uint64_t* offsets;
  uint32_t* sizes;
  uint64_t* total;
  long long clock_offset_ns;
  PushMsgWork w;
  // a PointCloud2 push's: the chain's parameters, and the device form's clouds and point counts of one chunk's slots
  const rpl_cloud_params* cloud;
  float* xyzi;
  uint32_t* points;
  // a LaserScan push that also projects its scans: the projection's parameters, the clouds' outputs, and the session's
  // tables of the projection (ScanCloudWork)
  const rpl_scan_cloud_params* proj;
  const rpl_msgs_out* clouds;
  unsigned long long* proj_carry;
  uint32_t* kept;
  const rpl::StreamMsgHeader* proj_hdr;  // RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS: the session's resolved headers, rows
  const float4* proj_xf;
  bool rescan;  // a re-gridding push: clouds are its re-grid messages (ChunkScanClouds::rescan)
  const rpl_msgs_out* merged;  // a merge push's merged scans, by group (nullptr: not a merge push)
};

// The host form's staging of a merge push (the session's mg_stage): the directory {fit end, total}, offsets and sizes,
// then the merged messages
struct MergeStage {
  unsigned long long *dir, *offsets;
  uint32_t* sizes;
  uint8_t* msgs;
};
MergeStage merge_stage_layout(Carve& k, uint32_t n_groups) {
  return MergeStage{k.take<unsigned long long>(2), k.take<unsigned long long>(n_groups), k.take<uint32_t>(n_groups),
                    k.take<uint8_t>(0)};
}

// The end of a merge push, once every chunk has held its grouped streams' grids (on st; the host form's lanes are
// drained): the directory over the groups and the merged messages, into the caller's arrays (dev) or staged in the
// session's mg_stage and copied back (the directory, then the messages that fit)
rpl_result rescan_merge_end(rpl_capsule_stream* cs, const PushMsgs& pm, bool dev, cudaStream_t st) {
  rpl_ctx* c = cs->c;
  const rpl_msgs_out& o = *pm.merged;
  const MergeTables t = merge_tables(cs);
  const uint32_t G = cs->mg_groups;
  rpl::RescanMergeArgs a{};
  a.members = t.members;
  a.begin = t.begin;
  a.max_age = t.max_age;
  a.n_groups = G;
  a.seq = cs->mg_seq + 1;
  a.row = t.row;
  a.held = t.held;
  a.rows = t.rows;
  a.hdr_scan = cs->msg_hdr;
  a.hdr_target = cs->xf_hdr;
  a.grid = cs->rescan;
  a.pick = t.pick;
  a.capacity = o.capacity;
  using u64 = unsigned long long;
  if (dev) {
    a.offsets = reinterpret_cast<u64*>(o.msg_offsets);
    a.sizes = o.msg_sizes;
    a.total = reinterpret_cast<u64*>(o.total_bytes);
    a.out = o.msgs;
  } else {
    Carve k{cs->mg_stage};
    const MergeStage m = merge_stage_layout(k, G);
    a.fit_end = m.dir;
    a.total = m.dir + 1;
    a.offsets = m.offsets;
    a.sizes = m.sizes;
    a.out = m.msgs;
  }
  RPL_CUDA(c, rpl::launch_rescan_merge(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches += G ? 2 : 1;
  if (dev) return RPL_RESULT_OK;
  u64 dir[2];  // {the end of the last message that fits, the total}
  RPL_CUDA(c, cudaMemcpyAsync(dir, a.fit_end, 16, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(o.msg_offsets, a.offsets, (size_t)G * 8, cudaMemcpyDeviceToHost, st),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(o.msg_sizes, a.sizes, (size_t)G * 4, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  *o.total_bytes = dir[1];
  if (dir[0]) RPL_CUDA(c, cudaMemcpy(o.msgs, a.out, dir[0], cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

// A push of the kind the entry point takes (bytes: a byte push); sp: a stamped one.  Host arrays (dev false, stream
// unused) run in the session's host chunks round-robin over the lanes, device arrays in its device chunks on `stream`.
// The arrays, sp's rx and scan_ts included, hold every stream.  pm: a message push, whose scans (pm->cloud: clouds) go
// into its messages (ranges, intensities, beam_counts and angle_increment unused).
rpl_result stream_push(rpl_capsule_stream* cs, const uint8_t* in, const uint32_t* counts, uint32_t sample_duration_us,
                       const rpl_scan_params* params, float* ranges, float* intensities, uint32_t* beam_counts,
                       float* angle_increment, uint32_t* scans_per_stream, const StampPush* sp, bool bytes, bool dev,
                       void* stream, const PushMsgs* pm = nullptr) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  cs->cloud_chunk = 0;
  if (!push_kind_ok(cs, bytes)) return RPL_RESULT_INVALID_DATA;
  if (!capsule_stream_args_ok(cs, in, counts, sample_duration_us, params, ranges, intensities, beam_counts,
                              scans_per_stream, pm != nullptr))
    return RPL_RESULT_INVALID_DATA;
  if (dev && !pm && !angle_increment && (params->flags & RPL_FLAG_PER_STREAM_FILTERS) != 0) {
    c->err = "a device push with RPL_FLAG_PER_STREAM_FILTERS needs angle_increment";
    return RPL_RESULT_INVALID_DATA;
  }
  const uint32_t chunk = dev ? cs->chunk_dev : cs->chunk_host;
  cudaStream_t st = nullptr;
  rpl_result r = RPL_RESULT_OK;
  if (dev) {
    if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
    RPL_CUDA(c, cudaStreamWaitEvent(st, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
    const size_t row = (size_t)cs->max_scans * cs->max_nodes;
    for (uint32_t s0 = 0; s0 < cs->n_streams && r == RPL_RESULT_OK; s0 += chunk) {
      const size_t so = (size_t)s0 * cs->max_scans;
      StampPush chunk_sp{};
      if (sp) {
        chunk_sp = *sp;
        chunk_sp.rx += (size_t)s0 * sp->stride_chunks;
        chunk_sp.scan_ts += so;
      }
      ChunkMsgs m{};
      if (pm) {  // straight into the caller's buffer and tables, one chunk after the other on st
        m.out = pm->msgs;
        m.first = s0 == 0;
        m.capacity = pm->capacity;
        m.carry = pm->w.carry;
        m.offsets = reinterpret_cast<unsigned long long*>(pm->offsets) + so;
        m.place = pm->w.place + so;
        m.total = reinterpret_cast<unsigned long long*>(pm->total);
        m.sizes = pm->sizes + so;
        m.hdr = cs->msg_hdr + s0;
        m.clock_offset_ns = pm->clock_offset_ns;
        m.cloud = pm->cloud;
        m.xyzi = pm->xyzi;
        m.points = pm->points;
        if (pm->proj)
          m.proj = ChunkScanClouds{pm->proj, pm->kept + so, pm->clouds->msgs, pm->clouds->capacity, pm->proj_carry,
                                   reinterpret_cast<unsigned long long*>(pm->clouds->msg_offsets) + so, nullptr,
                                   reinterpret_cast<unsigned long long*>(pm->clouds->total_bytes),
                                   pm->clouds->msg_sizes + so, nullptr, nullptr, pm->proj_hdr ? pm->proj_hdr + s0 : nullptr,
                                   pm->proj_xf ? pm->proj_xf + 3 * s0 : nullptr};
        if (pm->proj && pm->rescan)
          m.proj.rescan = rescan_chunk(cs, s0, std::min(chunk, cs->n_streams - s0), pm->merged != nullptr);
      }
      r = capsule_stream_chunk(c, c->lane[0], st, session_chunk(cs, s0, params, true, pm ? pm->cloud : nullptr),
                               std::min(chunk, cs->n_streams - s0), in + s0 * cs->in_stream, counts + s0,
                               sample_duration_us, params, pm ? nullptr : ranges + s0 * row,
                               pm ? nullptr : intensities + s0 * row, pm ? pm->w.beams + so : beam_counts + so,
                               pm ? pm->w.inc + so : angle_increment ? angle_increment + so : nullptr,
                               scans_per_stream + s0, sp ? &chunk_sp : nullptr, pm ? &m : nullptr);
    }
    if (r == RPL_RESULT_OK && pm && pm->merged) r = rescan_merge_end(cs, *pm, true, st);
  } else {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (counts[s] > cs->stride_in) {
        c->err = bytes ? "byte_counts[s] exceeds stride_bytes" : "capsule_counts[s] exceeds stride_capsules";
        return RPL_RESULT_INVALID_DATA;
      }
    RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
    for (int i = 0; i < kLanes; ++i) RPL_CUDA(c, cudaStreamWaitEvent(c->lane[i].stream, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
    HostMsgs hm{};
    if (pm) {
      uint32_t hdr_most = 0;
      for (const rpl::StreamMsgHeader& e : cs->msg_hdr_host) hdr_most = std::max(hdr_most, e.bytes);
      // a message's bytes at max_nodes, rounded up to 16 (PointCloud2: the tail, 16 B per point and is_dense)
      const size_t n = cs->max_nodes, most = pm->cloud ? (size_t)hdr_most + 116 + 16 * n + 1 : hdr_most + 32 + 8 * n + 4;
      const size_t bound = (most + 15) & ~(size_t)15;
      hm = HostMsgs{pm->msgs, pm->capacity, pm->offsets, pm->sizes, pm->total, (size_t)chunk * cs->max_scans * bound,
                    pm->clock_offset_ns, cs->msg_hdr, pm->w.carry, pm->w.place, cs->push_msg_extent,
                    cs->push_msg_extent_ready, cs->push_msg_dir_order, pm->cloud};
      if (pm->proj) {  // a projected cloud's bound: its message at max_nodes kept beams, rounded up to 16
        uint32_t proj_hdr_most = hdr_most;  // with transforms: the longest resolved header
        if (pm->proj_hdr) {
          proj_hdr_most = 0;
          for (const rpl::StreamMsgHeader& e : cs->xf_hdr_host) proj_hdr_most = std::max(proj_hdr_most, e.bytes);
        }
        uint32_t bins_most = 0;  // a re-gridding push's: the largest ranges_size
        for (const rpl_rescan_settings& e : cs->rescan_host)
          if (pm->rescan && e.enabled) bins_most = std::max(bins_most, rescan_bins(e));
        const size_t pmost = pm->rescan ? (size_t)proj_hdr_most + 36 + 4 * (size_t)bins_most
                                        : (size_t)proj_hdr_most + scan_cloud_tail_bytes(pm->proj->channels) +
                                              (size_t)scan_cloud_point_step(pm->proj->channels) * n + 1;
        hm.proj = pm->proj;
        hm.clouds = pm->clouds;
        hm.proj_chunk_bytes = (size_t)chunk * cs->max_scans * ((pmost + 15) & ~(size_t)15);
        hm.proj_carry = pm->proj_carry;
        hm.proj_extent_host = cs->push_scan_cloud_extent;
        hm.kept = pm->kept;
        hm.proj_dir_order = cs->push_scan_cloud_dir_order;
        hm.proj_hdr = pm->proj_hdr;
        hm.proj_xf = pm->proj_xf;
        if (pm->rescan) hm.rescan = cs;
        hm.merge = pm->merged != nullptr;
      }
    }
    const HostWire h{in, counts, cs->in_stream, sample_duration_us, cs->max_nodes, cs->max_scans, params, ranges,
                     intensities, angle_increment, beam_counts, scans_per_stream, sp, sp ? sp->stride_chunks : 0u,
                     pm ? &hm : nullptr};
    r = push_host(c, h, cs->n_streams, chunk,
                  [&](Carve&, uint32_t s0) { return session_chunk(cs, s0, params, false, pm ? pm->cloud : nullptr); });
    if (r == RPL_RESULT_OK && pm && pm->merged) r = rescan_merge_end(cs, *pm, false, c->lane[0].stream);
  }
  cs->parity ^= 1u;
  cs->prev_stamped = cs->carry_stamped = sp != nullptr;
  if (dev) RPL_CUDA(c, cudaEventRecord(cs->done, st), RPL_RESULT_OPERATION_FAIL);
  if (r == RPL_RESULT_OK) {
    cs->cloud_chunk = chunk;
    cs->cloud_arena = cs->parity ^ 1u;
  }
  return r;
}

// the parameter rules of the PointCloud2 chain (rpl_cloud_batch_dev and the session clouds)
bool cloud_params_ok(rpl_ctx* c, const rpl_cloud_params* p) {
  if (p->sor_k > 32) {
    c->err = "sor_k > 32";
    return false;
  }
  if (p->voxel_size != 0.0f && !(p->voxel_size >= 1e-6f && p->range_max < 1000.0f)) {
    c->err = "voxel grid: voxel_size must be >= 1e-6 m and range_max < 1000 m (cell indices must fit 31 bits)";
    return false;
  }
  return true;
}

// a cloud call's chain rules: its params', or with RPL_CLOUD_PER_STREAM_CHAIN those of the session's resolved table
bool cloud_call_ok(rpl_capsule_stream* cs, const rpl_cloud_params* p) {
  rpl_ctx* c = cs->c;
  if ((p->flags & RPL_CLOUD_PER_STREAM_FOOTPRINTS) != 0 && cs->footprints_host.empty()) {
    c->err = "per-stream cloud footprints requested before rpl_capsule_stream_set_scan_footprints set every stream";
    return false;
  }
  if ((p->flags & RPL_CLOUD_PER_STREAM_CHAIN) == 0) return cloud_params_ok(c, p);
  if (cs->clouds_host.empty()) {
    c->err = "per-stream clouds requested before rpl_capsule_stream_set_clouds set every stream";
    return false;
  }
  if (!cs->clouds_bad.empty()) {
    c->err = cs->clouds_bad;
    return false;
  }
  return true;
}

// The scans of streams [s0, s0 + ns) of the session's last push, one chunk of that push, as the scan kernels read
// them: the chunk's region of the push's arena, its slots' views (which count from node 0 of stream s0 there) and
// the holder's capacity as the stride.
rpl::ScanBatchArgs last_push_scans(const rpl_capsule_stream* cs, uint32_t s0, uint32_t ns) {
  rpl::ScanBatchArgs a{};
  a.nodes = reinterpret_cast<const uint2*>(cs->arena[cs->cloud_arena] + (size_t)s0 * cs->stride_nodes);
  a.views = reinterpret_cast<const uint2*>(cs->views + (size_t)s0 * cs->max_scans);
  a.counts = reinterpret_cast<const uint32_t*>(a.views);
  a.nodes_total = (unsigned long long)ns * cs->stride_nodes;
  a.n_scans = ns * cs->max_scans;
  a.stride = cs->max_nodes;
  return a;
}

bool stream_cloud_args_ok(rpl_capsule_stream* cs, const rpl_cloud_params* params, float* xyzi, uint32_t* point_counts) {
  rpl_ctx* c = cs->c;
  if (!params || !xyzi || !point_counts) {
    c->err = "null params, xyzi or point_counts";
    return false;
  }
  if (!cloud_call_ok(cs, params)) return false;
  if ((params->flags & RPL_CLOUD_PER_STREAM) != 0 && !lidars_ok(cs)) return false;
  if (cs->cloud_chunk == 0) {
    c->err = "no clouds to take: the session has not pushed yet, or its last push failed";
    return false;
  }
  return true;
}

// grows the session's message work block (an earlier messages call, on any stream, may still read it)
rpl_result grow_msg_work(rpl_capsule_stream* cs, size_t bytes) {
  rpl_ctx* c = cs->c;
  if (cs->msg_work_bytes >= bytes) return RPL_RESULT_OK;
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);
  cudaFree(cs->msg_work);
  cs->msg_work = nullptr;
  cs->msg_work_bytes = 0;
  RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&cs->msg_work), bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
  cs->msg_work_bytes = bytes;
  return RPL_RESULT_OK;
}

// The device form of a call on the last push: once the device is entered and the message work block has grown to
// msg_work bytes (0: the call uses none), fn(st) enqueues the call on `stream` (NULL: lane 0's) behind the last push's
// kernels, which are done before it reads the push's arena and views; the session's next push waits for it.
template <class F>
rpl_result last_push_dev(rpl_capsule_stream* cs, void* stream, size_t msg_work, F fn) {
  rpl_ctx* c = cs->c;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  if (const rpl_result r = grow_msg_work(cs, msg_work); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamWaitEvent(st, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
  const rpl_result r = fn(st);
  RPL_CUDA(c, cudaEventRecord(cs->done, st), RPL_RESULT_OPERATION_FAIL);
  return r;
}

rpl_result stream_cloud_dev(rpl_capsule_stream* cs, const rpl_cloud_params* params, float* xyzi,
                            uint32_t* point_counts, void* stream) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  if (!stream_cloud_args_ok(cs, params, xyzi, point_counts)) return RPL_RESULT_INVALID_DATA;
  const size_t row = (size_t)cs->max_scans * cs->max_nodes * 4;
  return last_push_dev(cs, stream, 0, [&](cudaStream_t st) -> rpl_result {
    rpl_result r = RPL_RESULT_OK;
    for (uint32_t s0 = 0; s0 < cs->n_streams && r == RPL_RESULT_OK; s0 += cs->cloud_chunk) {
      const uint32_t ns = std::min(cs->cloud_chunk, cs->n_streams - s0);
      const rpl::ScanFootprint* fp = cloud_footprints_at(cs, params, s0, ns);
      r = stream_cloud_chunk(cs->c, cs->c->lane[0], last_push_scans(cs, s0, ns), lidars_at(cs, s0),
                             chains_at(cs, s0, fp != nullptr), cs->max_scans, params, xyzi + (size_t)s0 * row,
                             point_counts + (size_t)s0 * cs->max_scans, st, fp);
    }
    return r;
  });
}

// the host variant: the last push's chunks round-robin over the lanes, each lane's clouds staged in its block and
// copied back while the next chunk runs on the other lane
rpl_result stream_cloud(rpl_capsule_stream* cs, const rpl_cloud_params* params, float* xyzi, uint32_t* point_counts) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!stream_cloud_args_ok(cs, params, xyzi, point_counts)) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  const uint32_t chunk = cs->cloud_chunk;
  const size_t NS = (size_t)chunk * cs->max_scans, row = (size_t)cs->max_scans * cs->max_nodes * 4;
  struct Regions {
    float* xyzi;
    uint32_t* counts;
  };
  auto layout = [&](Carve& k) { return Regions{k.take<float>(NS * cs->max_nodes * 4), k.take<uint32_t>(NS)}; };
  if (const rpl_result r = grow_stage(c, kLanes, layout); r != RPL_RESULT_OK) return r;
  for (int i = 0; i < kLanes; ++i) RPL_CUDA(c, cudaStreamWaitEvent(c->lane[i].stream, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
  const cudaMemcpyKind d2h = cudaMemcpyDeviceToHost;
  auto run_chunk = [&](Lane& l, uint32_t s0, uint32_t ns) -> rpl_result {
    Carve k{l.stage};
    const Regions d = layout(k);
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);  // the lane's previous chunk has left
    const rpl::ScanFootprint* fp = cloud_footprints_at(cs, params, s0, ns);
    const rpl_result r = stream_cloud_chunk(c, l, last_push_scans(cs, s0, ns), lidars_at(cs, s0),
                                            chains_at(cs, s0, fp != nullptr), cs->max_scans, params, d.xyzi, d.counts,
                                            l.stream, fp);
    if (r != RPL_RESULT_OK) return r;
    RPL_CUDA(c, cudaMemcpyAsync(xyzi + (size_t)s0 * row, d.xyzi, ns * row * 4, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemcpyAsync(point_counts + (size_t)s0 * cs->max_scans, d.counts, (size_t)ns * cs->max_scans * 4, d2h,
                                l.stream),
             RPL_RESULT_OPERATION_FAIL);
    return RPL_RESULT_OK;
  };
  return run_chunks(c, cs->n_streams, chunk, run_chunk);
}

// ---- packed LaserScan / PointCloud2 messages of the last push (DESIGN.md 5.9) -------------------------------------
// Per call: the scan kernels (LaserScan) or the session cloud chain (PointCloud2) over the last push's views into the
// session's work block, the sizes and offsets pass over every slot, then the writers.  The device form writes every
// message into the caller's buffer; the host form reads the tables back first and then writes and copies the
// messages chunk by chunk over the lanes, so that only message bytes cross the link.

// The device table of the per-stream clouds from the entries as set and the frames' range_max, with its summary: each
// stream's route (the fusion guard of launch_fast at its resolved range_max) and why a flagged call would fail.  The
// caller has passed cs->done.
rpl_result clouds_resolve(rpl_capsule_stream* cs, const std::vector<rpl_scan_footprint>* footprints = nullptr) {
  rpl_ctx* c = cs->c;
  const std::vector<rpl_scan_footprint>& fps = footprints ? *footprints : cs->footprints_host;
  std::vector<rpl::CloudSettings> t(cs->n_streams);
  uint32_t routes = 0, sor_k = 0;
  bool voxel = false;
  std::string bad;
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    const rpl_cloud_settings& e = cs->clouds_host[s];
    rpl::CloudSettings& d = t[s];
    d.range_min = e.range_min;
    d.range_max = e.range_max != 0.0f ? e.range_max : cs->msg_hdr_host[s].range_max;
    d.intensity_min = e.intensity_min;
    d.voxel = e.voxel_size;
    d.sor_k = e.sor_k;
    d.sor_alpha = e.sor_alpha;
    if (!e.enabled) {
      d.route = rpl::kCloudOff;
    } else if (e.sor_k == 0 && e.voxel_size == 0.0f) {
      d.route = rpl::kCloudWindow;
    } else {
      if (e.voxel_size != 0.0f && !(d.range_max < 1000.0f) && bad.empty())
        bad = "voxel grid: a stream's range_max, resolved against rpl_capsule_stream_set_frames, must be < 1000 m";
      const bool fusable = e.voxel_size == 0.0f || (e.voxel_size <= 4.0f && d.range_max / e.voxel_size < 32000.0f);
      d.route = fusable ? rpl::kCloudFused : rpl::kCloudSeparate;
      sor_k = std::max(sor_k, e.sor_k);
      voxel = voxel || e.voxel_size > 0.0f;
    }
    routes |= 1u << d.route;
  }
  RPL_CUDA(c, cudaMemcpy(cs->clouds, t.data(), t.size() * sizeof(rpl::CloudSettings), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  // the footprint table: a stream with a polygon is never fused (its SOR / voxel grid run behind the footprint pass)
  uint32_t routes_fp = 0;
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (t[s].route == rpl::kCloudFused && !fps.empty() && has_polygons(fps[s])) t[s].route = rpl::kCloudSeparate;
    routes_fp |= 1u << t[s].route;
  }
  RPL_CUDA(c, cudaMemcpy(cs->clouds_fp, t.data(), t.size() * sizeof(rpl::CloudSettings), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->cloud_routes_fp = routes_fp;
  cs->cloud_routes = routes;
  cs->cloud_sor_k = sor_k;
  cs->cloud_voxel = voxel;
  cs->clouds_bad = bad;
  return RPL_RESULT_OK;
}

// The device tables of the per-stream transforms from entries t and target frames f: each stream's rows and its
// clouds' header (a disabled entry's the LaserScan's).  The caller has passed cs->done and made the tables.
rpl_result transforms_resolve(rpl_capsule_stream* cs, const std::vector<rpl_scan_cloud_transform>& t,
                              const std::vector<std::string>& f) {
  rpl_ctx* c = cs->c;
  std::vector<float4> rows(3 * (size_t)cs->n_streams);
  std::vector<rpl::StreamMsgHeader> h(cs->n_streams);
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    scan_cloud_rows(t[s], &rows[3 * (size_t)s]);
    h[s] = t[s].enabled ? msg_header(f[s].data(), f[s].size(), cs->msg_hdr_host[s].range_max) : cs->msg_hdr_host[s];
  }
  RPL_CUDA(c, cudaMemcpy(cs->xf, rows.data(), rows.size() * sizeof(float4), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpy(cs->xf_hdr, h.data(), h.size() * sizeof(rpl::StreamMsgHeader), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->xf_hdr_host = std::move(h);
  return RPL_RESULT_OK;
}

// Empties the held grids of the merge groups' streams `mask` takes in (nullptr: all), on `st`, when there are groups
rpl_result merges_empty(rpl_capsule_stream* cs, const uint8_t* mask, cudaStream_t st) {
  if (!cs->mg_block) return RPL_RESULT_OK;
  rpl::RescanHeld* held = merge_tables(cs).held;
  for (uint32_t s = 0; s < cs->n_streams;) {
    if (mask && !mask[s]) {
      ++s;
      continue;
    }
    uint32_t e = s + 1;
    while (e < cs->n_streams && (!mask || mask[e])) ++e;
    RPL_CUDA(cs->c, cudaMemsetAsync(held + s, 0, (size_t)(e - s) * sizeof(rpl::RescanHeld), st),
             RPL_RESULT_OPERATION_FAIL);
    s = e;
  }
  return RPL_RESULT_OK;
}

// the transforms of the projected clouds: the masked entries and target frames replace the table's, all or none
rpl_result stream_set_scan_cloud_transforms(rpl_capsule_stream* cs, const rpl_scan_cloud_transform* transforms,
                                            const char* const* target_frames, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!transforms || !target_frames) {
    c->err = "null transforms or target_frames";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_scan_cloud_transform> t = cs->xf_host;
  std::vector<std::string> f = cs->xf_frames;
  if (t.empty()) {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_capsule_stream_set_scan_cloud_transforms call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
    f.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    const bool on = transforms[s].enabled != 0;
    if (on && !scan_cloud_transform_ok(c, transforms[s], target_frames[s], true)) return RPL_RESULT_INVALID_DATA;
    t[s] = transforms[s];
    f[s] = on ? std::string(target_frames[s]) : std::string();
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->xf) RPL_CUDA(c, dev_alloc(&cs->xf, 3 * (size_t)cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  if (!cs->xf_hdr) RPL_CUDA(c, dev_alloc(&cs->xf_hdr, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a messages call may still read them
  if (const rpl_result r = transforms_resolve(cs, t, f); r != RPL_RESULT_OK) return r;
  if (const rpl_result r = merges_empty(cs, stream_mask, c->lane[0].stream); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamSynchronize(c->lane[0].stream), RPL_RESULT_OPERATION_FAIL);
  cs->xf_host = std::move(t);
  cs->xf_frames = std::move(f);
  return RPL_RESULT_OK;
}

// Empties the windows of the streams `mask` takes in (nullptr: all), on `st`: one clear per run of them
rpl_result windows_empty(rpl_capsule_stream* cs, const uint8_t* mask, cudaStream_t st) {
  for (uint32_t s = 0; s < cs->n_streams;) {
    if (mask && !mask[s]) {
      ++s;
      continue;
    }
    uint32_t e = s + 1;
    while (e < cs->n_streams && (!mask || mask[e])) ++e;
    RPL_CUDA(cs->c, cudaMemsetAsync(cs->win_state + s, 0, (size_t)(e - s) * sizeof(uint2), st), RPL_RESULT_OPERATION_FAIL);
    s = e;
  }
  return RPL_RESULT_OK;
}

// Lays the windows out from the re-grid entries t and the windows w as the set call will leave them, once cs->done has
// passed: each enabled stream with observations >= 2 gets (observations - 1) * ranges_size floats of a new ring.  The
// streams `mask` leaves out (their entries and so their sizes unchanged) keep their window, copied; the others start
// empty.  Running out of memory changes nothing.
rpl_result windows_layout(rpl_capsule_stream* cs, const std::vector<rpl_rescan_settings>& t,
                          const std::vector<rpl_rescan_window>& w, const uint8_t* mask) {
  rpl_ctx* c = cs->c;
  const uint32_t n = cs->n_streams;
  std::vector<rpl::RescanWindow> win(n);
  std::vector<uint32_t> streams;
  unsigned long long total = 0;
  for (uint32_t s = 0; s < n; ++s) {
    const uint32_t bins = t.empty() || !t[s].enabled ? 0u : rescan_bins(t[s]);
    const bool windowed = bins > 0 && w[s].observations > 1;
    win[s] = rpl::RescanWindow{total, w[s].observations, w[s].statistic};
    if (windowed) {
      streams.push_back(s);
      total += (unsigned long long)(w[s].observations - 1) * bins;
    }
  }
  if (!cs->win) {  // the first call: the per-stream tables, every window empty; all three or none
    rpl::RescanWindow* win = nullptr;
    uint32_t* streams_d = nullptr;
    uint2* state = nullptr;
    cudaError_t e = dev_alloc(&win, n);
    if (e == cudaSuccess) e = dev_alloc(&streams_d, n);
    if (e == cudaSuccess) e = dev_alloc(&state, n);
    if (e == cudaSuccess) e = cudaMemset(state, 0, (size_t)n * sizeof(uint2));
    if (e != cudaSuccess) {
      cudaFree(win);
      cudaFree(streams_d);
      cudaFree(state);
      RPL_CUDA(c, e, e == cudaErrorMemoryAllocation ? RPL_RESULT_INSUFFICIENT_MEMORY : RPL_RESULT_OPERATION_FAIL);
    }
    cs->win = win;
    cs->win_streams = streams_d;
    cs->win_state = state;
  }
  float* ring = nullptr;
  if (total) RPL_CUDA(c, dev_alloc(&ring, total), RPL_RESULT_INSUFFICIENT_MEMORY);
  std::vector<uint8_t> kept(n, 0);  // a stream with a window in both layouts that the call leaves out
  for (uint32_t s : cs->win_streams_host) kept[s] = mask && !mask[s] ? 1 : 0;
  cudaError_t e = cudaSuccess;
  for (uint32_t s : streams)
    if (kept[s] && e == cudaSuccess)
      e = cudaMemcpy(ring + win[s].ring, cs->win_ring + cs->win_layout_host[s].ring,
                     (size_t)(w[s].observations - 1) * rescan_bins(t[s]) * 4, cudaMemcpyDeviceToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(cs->win, win.data(), (size_t)n * sizeof(rpl::RescanWindow), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && !streams.empty())
    e = cudaMemcpy(cs->win_streams, streams.data(), streams.size() * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(ring);
    RPL_CUDA(c, e, RPL_RESULT_OPERATION_FAIL);
  }
  if (const rpl_result r = windows_empty(cs, mask, c->lane[0].stream); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamSynchronize(c->lane[0].stream), RPL_RESULT_OPERATION_FAIL);
  cudaFree(cs->win_ring);
  cs->win_ring = ring;
  cs->win_layout_host = std::move(win);
  cs->win_streams_host = std::move(streams);
  return RPL_RESULT_OK;
}

// the windows over the re-gridded scans: the masked entries of `windows` replace the table's, all or none
rpl_result stream_set_rescan_windows(rpl_capsule_stream* cs, const rpl_rescan_window* windows, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!windows) {
    c->err = "null windows";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_rescan_window> w = cs->win_host;
  if (w.empty()) w.assign(cs->n_streams, rpl_rescan_window{1u, RPL_RESCAN_WINDOW_MEDIAN});
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    if (!rescan_window_ok(c, windows[s])) return RPL_RESULT_INVALID_DATA;
    w[s] = windows[s];
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push may still read them
  if (const rpl_result r = windows_layout(cs, cs->rescan_host, w, stream_mask); r != RPL_RESULT_OK) return r;
  if (const rpl_result r = merges_empty(cs, stream_mask, c->lane[0].stream); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamSynchronize(c->lane[0].stream), RPL_RESULT_OPERATION_FAIL);
  cs->win_host = std::move(w);
  return RPL_RESULT_OK;
}

// the merge groups: a new layout replaces the old whole, every held grid empty, all or none
rpl_result stream_set_rescan_merges(rpl_capsule_stream* cs, const uint32_t* group_of_stream, const uint32_t* max_age,
                                    uint32_t n_groups) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!group_of_stream || (n_groups && !max_age)) {
    c->err = "null group_of_stream or max_age";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_groups > cs->n_streams) {
    c->err = "n_groups exceeds n_streams";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<uint32_t> count(n_groups, 0), streams, row(cs->n_streams, rpl::kRescanMergeNone);
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    const uint32_t g = group_of_stream[s];
    if (g == rpl::kRescanMergeNone) continue;
    if (g >= n_groups) {
      c->err = "a group index must be below n_groups or RPL_RESCAN_MERGE_NONE";
      return RPL_RESULT_INVALID_DATA;
    }
    count[g]++;
    row[s] = (uint32_t)streams.size();
    streams.push_back(s);
  }
  for (uint32_t g = 0; g < n_groups; ++g) {
    if (count[g] == 0) {
      c->err = "every merge group needs a member";
      return RPL_RESULT_INVALID_DATA;
    }
    if (max_age[g] > 65535) {
      c->err = "max_age must be at most 65535";
      return RPL_RESULT_INVALID_DATA;
    }
  }
  std::vector<uint32_t> begin(n_groups + 1, 0), members(streams.size());
  for (uint32_t g = 0; g < n_groups; ++g) begin[g + 1] = begin[g] + count[g];
  std::vector<uint32_t> at(begin.begin(), begin.end() - 1);
  for (uint32_t s : streams) members[at[group_of_stream[s]]++] = s;  // ascending within each group
  const uint32_t ng = (uint32_t)streams.size();
  Carve k;
  merge_tables_layout(k, cs->n_streams, ng, n_groups);
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  unsigned char* block = nullptr;
  RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&block), k.bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
  Carve kb{block};
  const MergeTables t = merge_tables_layout(kb, cs->n_streams, ng, n_groups);
  cudaError_t e = cudaMemcpy(t.row, row.data(), row.size() * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(t.held, 0, (size_t)cs->n_streams * sizeof(rpl::RescanHeld));
  if (e == cudaSuccess && ng) e = cudaMemcpy(t.streams, streams.data(), (size_t)ng * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && ng) e = cudaMemcpy(t.members, members.data(), (size_t)ng * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t.begin, begin.data(), begin.size() * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && n_groups) e = cudaMemcpy(t.max_age, max_age, (size_t)n_groups * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(block);
    RPL_CUDA(c, e, RPL_RESULT_OPERATION_FAIL);
  }
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push may still read the old block
  cudaFree(cs->mg_block);
  cs->mg_block = block;
  cs->mg_set = true;
  cs->mg_groups = n_groups;
  cs->mg_members_host = std::move(members);
  cs->mg_begin_host = std::move(begin);
  cs->mg_streams_host = std::move(streams);
  return RPL_RESULT_OK;
}

// the re-gridded scans' entries: the masked entries of `settings` replace the table's, all or none
rpl_result stream_set_rescans(rpl_capsule_stream* cs, const rpl_rescan_settings* settings, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!settings) {
    c->err = "null settings";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_rescan_settings> t = cs->rescan_host;
  if (t.empty()) {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_capsule_stream_set_rescans call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    if (settings[s].enabled && !rescan_ok(c, settings[s])) return RPL_RESULT_INVALID_DATA;
    t[s] = settings[s];
  }
  std::vector<rpl::RescanGrid> g(cs->n_streams);
  std::vector<uint32_t> bins(cs->n_streams);
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    g[s] = rescan_grid(t[s], true);
    bins[s] = g[s].bins;
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->rescan) RPL_CUDA(c, dev_alloc(&cs->rescan, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  if (!cs->rescan_bins) RPL_CUDA(c, dev_alloc(&cs->rescan_bins, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a messages call may still read them
  if (!cs->win_host.empty())  // the masked streams' grids may change: their windows start over
    if (const rpl_result r = windows_layout(cs, t, cs->win_host, stream_mask); r != RPL_RESULT_OK) return r;
  if (const rpl_result r = merges_empty(cs, stream_mask, c->lane[0].stream); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamSynchronize(c->lane[0].stream), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpy(cs->rescan, g.data(), g.size() * sizeof(rpl::RescanGrid), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpy(cs->rescan_bins, bins.data(), bins.size() * 4, cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->rescan_host = std::move(t);
  return RPL_RESULT_OK;
}

rpl_result stream_set_frames(rpl_capsule_stream* cs, const char* const* frame_ids, const float* range_max) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!frame_ids) {
    c->err = "null frame_ids";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl::StreamMsgHeader> h(cs->n_streams);
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (!frame_ids[s]) {
      c->err = "null frame_ids[s]";
      return RPL_RESULT_INVALID_DATA;
    }
    const size_t L = std::strlen(frame_ids[s]);
    if (!frame_id_length_ok(c, L)) return RPL_RESULT_INVALID_DATA;
    h[s] = msg_header(frame_ids[s], L, range_max ? range_max[s] : cs->msg_hdr_host[s].range_max);
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a messages call may still read them
  RPL_CUDA(c, cudaMemcpy(cs->msg_hdr, h.data(), h.size() * sizeof(rpl::StreamMsgHeader), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->msg_hdr_host = std::move(h);
  if (const rpl_result r = merges_empty(cs, nullptr, c->lane[0].stream); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaStreamSynchronize(c->lane[0].stream), RPL_RESULT_OPERATION_FAIL);
  if (!cs->xf_host.empty())  // a disabled transform entry's header follows the frames
    if (const rpl_result r = transforms_resolve(cs, cs->xf_host, cs->xf_frames); r != RPL_RESULT_OK) return r;
  return cs->clouds_host.empty() ? RPL_RESULT_OK : clouds_resolve(cs);  // a range_max of 0 follows the frames
}

// the per-stream lidar settings: the masked entries of `settings` replace the table's, all or none
rpl_result stream_set_lidars(rpl_capsule_stream* cs, const rpl_lidar_settings* settings, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!settings) {
    c->err = "null settings";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl::LidarSettings> t = cs->lidars_host;
  if (t.empty()) {  // the first call sets every stream: no stream is left without a sample duration
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_*_stream_set_lidars call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    // the decoders divide by it (the angular-jump threshold)
    if (!sample_duration_ok(c, settings[s].timing.sample_duration_us)) return RPL_RESULT_INVALID_DATA;
    std::memcpy(&t[s], &settings[s], sizeof(rpl::LidarSettings));
  }
  uint32_t modes = 0;
  for (const rpl::LidarSettings& e : t) modes |= e.mode_a ? 2u : 1u;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->lidars)
    RPL_CUDA(c, dev_alloc(&cs->lidars, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push or messages call may still read it
  RPL_CUDA(c, cudaMemcpy(cs->lidars, t.data(), t.size() * sizeof(rpl::LidarSettings), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->lidars_host = std::move(t);
  cs->lidar_modes = modes;
  return RPL_RESULT_OK;
}

// the per-stream clouds: the masked entries of `settings` replace the table's, all or none
rpl_result stream_set_clouds(rpl_capsule_stream* cs, const rpl_cloud_settings* settings, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!settings) {
    c->err = "null settings";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_cloud_settings> t = cs->clouds_host;
  if (t.empty()) {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_capsule_stream_set_clouds call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    rpl_cloud_params p{};
    std::memcpy(&p, &settings[s], offsetof(rpl_cloud_params, is_new_protocol));  // the chain's six fields
    if (!cloud_params_ok(c, &p)) return RPL_RESULT_INVALID_DATA;
    t[s] = settings[s];
  }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->clouds) RPL_CUDA(c, dev_alloc(&cs->clouds, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  if (!cs->clouds_fp) RPL_CUDA(c, dev_alloc(&cs->clouds_fp, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a cloud or messages call may still read it
  cs->clouds_host = std::move(t);
  return clouds_resolve(cs);
}

// the per-stream LaserScan filters: the masked entries of `settings` replace the table's, all or none
rpl_result stream_set_scan_filters(rpl_capsule_stream* cs, const rpl_scan_filter_settings* settings,
                                   const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!settings) {
    c->err = "null settings";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_scan_filter_settings> t = cs->filters_host;
  if (t.empty()) {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_capsule_stream_set_scan_filters call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    if (!scan_filter_ok(c, settings[s])) return RPL_RESULT_INVALID_DATA;
    t[s] = settings[s];
  }
  std::vector<rpl::ScanFilter> d(cs->n_streams);
  for (uint32_t s = 0; s < cs->n_streams; ++s) d[s] = scan_filter_entry(t[s]);
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->filters) RPL_CUDA(c, dev_alloc(&cs->filters, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push or messages call may still read it
  RPL_CUDA(c, cudaMemcpy(cs->filters, d.data(), d.size() * sizeof(rpl::ScanFilter), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->filters_host = std::move(t);
  return RPL_RESULT_OK;
}

// the per-stream footprints: the masked entries of `footprints` replace the table's, all or none
rpl_result stream_set_scan_footprints(rpl_capsule_stream* cs, const rpl_scan_footprint* footprints,
                                      const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!footprints) {
    c->err = "null footprints";
    return RPL_RESULT_INVALID_DATA;
  }
  std::vector<rpl_scan_footprint> t = cs->footprints_host;
  if (t.empty()) {
    for (uint32_t s = 0; s < cs->n_streams; ++s)
      if (stream_mask && !stream_mask[s]) {
        c->err = "the first rpl_capsule_stream_set_scan_footprints call must set every stream";
        return RPL_RESULT_INVALID_DATA;
      }
    t.resize(cs->n_streams);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    if (stream_mask && !stream_mask[s]) continue;
    if (!scan_footprint_ok(c, footprints[s])) return RPL_RESULT_INVALID_DATA;
    t[s] = footprints[s];
  }
  std::vector<rpl::ScanFootprint> d(cs->n_streams);
  for (uint32_t s = 0; s < cs->n_streams; ++s) d[s] = scan_footprint_entry(t[s]);
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  if (!cs->footprints) RPL_CUDA(c, dev_alloc(&cs->footprints, cs->n_streams), RPL_RESULT_INSUFFICIENT_MEMORY);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push or messages call may still read it
  // the clouds' footprint route table follows the new footprints (every allocation is made before the tables change)
  if (!cs->clouds_host.empty())
    if (const rpl_result r = clouds_resolve(cs, &t); r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaMemcpy(cs->footprints, d.data(), d.size() * sizeof(rpl::ScanFootprint), cudaMemcpyHostToDevice),
           RPL_RESULT_OPERATION_FAIL);
  cs->footprints_host = std::move(t);
  return RPL_RESULT_OK;
}

// the PointCloud2 members between the header and the data: the fields x, y, z, intensity (float32), point_step 16
rpl::CloudTail cloud_tail() {
  const char* names[4] = {"x", "y", "z", "intensity"};
  const uint8_t types[4] = {7, 7, 7, 7};  // FLOAT32
  return pointcloud2_tail<rpl::CloudTail>(names, types, 4, 16);
}

// the work block of a messages call: scan outputs of every slot (LaserScan ranges then intensities, or xyzi), their
// counts and angle increments; the host form's tables behind them
struct MsgWork {
  float* data;
  uint32_t* counts;
  float* inc;
  unsigned long long* offsets;
  uint32_t* sizes;
  unsigned long long* total;
  uint32_t* kept;  // kScanCloud: the projections' point counts
};
MsgWork msg_work_layout(const rpl_capsule_stream* cs, rpl::MsgKind kind, bool tables, Carve& k) {
  const size_t NS = (size_t)cs->n_streams * cs->max_scans;
  const size_t floats = NS * cs->max_nodes * (kind == rpl::MsgKind::kPointCloud2 ? 4 : 2);
  return MsgWork{k.take<float>(floats), k.take<uint32_t>(NS), k.take<float>(NS),
                 k.take<unsigned long long>(tables ? NS : 0), k.take<uint32_t>(tables ? NS : 0),
                 k.take<unsigned long long>(tables ? 1 : 0), k.take<uint32_t>(kind == rpl::MsgKind::kScanCloud ? NS : 0)};
}

// the params of a kScanCloud or kRescan messages call
struct ScanCloudCall {
  const rpl_scan_params* scan;
  const rpl_scan_cloud_params* cloud;
};

// a kScanCloud or kRescan messages call with RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS
bool scan_cloud_transforms(const void* params) {
  return (static_cast<const ScanCloudCall*>(params)->cloud->channels & rpl::kScanCloudPerStreamTransforms) != 0;
}

// the LaserScan params of a messages call (kLaserScan, kScanCloud, kRescan), nullptr for kPointCloud2
const rpl_scan_params* msgs_scan_params(rpl::MsgKind kind, const void* params) {
  if (kind == rpl::MsgKind::kLaserScan) return static_cast<const rpl_scan_params*>(params);
  if (kind == rpl::MsgKind::kScanCloud || kind == rpl::MsgKind::kRescan)
    return static_cast<const ScanCloudCall*>(params)->scan;
  return nullptr;
}

// the rules of a session projection's params: the channels, and RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS (with which the
// viewpoint is accepted) only after the first set_scan_cloud_transforms
bool scan_cloud_call_ok(rpl_capsule_stream* cs, const rpl_scan_cloud_params& p) {
  const bool xf = (p.channels & rpl::kScanCloudPerStreamTransforms) != 0;
  if (!scan_cloud_ok(cs->c, p, rpl::kScanCloudPerStreamTransforms | (xf ? rpl::kScanCloudViewpoint : 0u))) return false;
  if (xf && cs->xf_host.empty()) {
    cs->c->err = "RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS before the first rpl_capsule_stream_set_scan_cloud_transforms";
    return false;
  }
  return true;
}

bool stream_msgs_args_ok(rpl_capsule_stream* cs, rpl::MsgKind kind, const void* params, const void* msgs,
                         const void* offsets, const void* sizes, const void* total, bool dev) {
  rpl_ctx* c = cs->c;
  if (!params || !msgs || !offsets || !sizes || !total) {
    c->err = "null params, msgs, msg_offsets, msg_sizes or total_bytes";
    return false;
  }
  if (kind == rpl::MsgKind::kPointCloud2 && !cloud_call_ok(cs, static_cast<const rpl_cloud_params*>(params)))
    return false;
  if (kind == rpl::MsgKind::kScanCloud || kind == rpl::MsgKind::kRescan) {
    const auto* q = static_cast<const ScanCloudCall*>(params);
    if (!q->scan || !q->cloud) {
      c->err = "null scan_params or cloud_params";
      return false;
    }
    if (!scan_cloud_call_ok(cs, *q->cloud)) return false;
    if (kind == rpl::MsgKind::kRescan && cs->rescan_host.empty()) {
      c->err = "rescan_msgs before the first rpl_capsule_stream_set_rescans";
      return false;
    }
  }
  const rpl_scan_params* sp = msgs_scan_params(kind, params);
  const bool per_stream = sp ? (sp->flags & RPL_FLAG_PER_STREAM) != 0
                             : (static_cast<const rpl_cloud_params*>(params)->flags & RPL_CLOUD_PER_STREAM) != 0;
  if (per_stream && !lidars_ok(cs)) return false;
  if (sp && (sp->flags & RPL_FLAG_PER_STREAM_FILTERS) != 0 && !filters_ok(cs)) return false;
  if (dev && ((reinterpret_cast<uintptr_t>(msgs) & 15u) || misaligned8(offsets) || misaligned8(total) ||
              (reinterpret_cast<uintptr_t>(sizes) & 3u))) {
    c->err = "msgs must be 16-byte aligned, msg_offsets and total_bytes 8-byte, msg_sizes 4-byte aligned";
    return false;
  }
  if (cs->cloud_chunk == 0) {
    c->err = "no messages to take: the session has not pushed yet, or its last push failed";
    return false;
  }
  return true;
}

// the projection of every slot's LaserScan in w (kScanCloud, kRescan): the count pass's arguments over all slots
// (msgs_write adds the placement)
rpl::ScanCloudArgs scan_cloud_msg_args(const rpl_capsule_stream* cs, const void* params, const MsgWork& w) {
  const auto* q = static_cast<const ScanCloudCall*>(params);
  const size_t NS = (size_t)cs->n_streams * cs->max_scans;
  rpl::ScanCloudArgs a{};
  scan_cloud_setup(a, *q->cloud);
  a.m.hdr = cs->msg_hdr;
  a.m.counts = w.counts;
  a.m.ranges = w.data;
  a.m.intensities = w.data + NS * cs->max_nodes;
  a.m.angle_increment = w.inc;
  a.m.stride = cs->max_nodes;
  a.m.max_scans = cs->max_scans;
  a.m.n = (uint32_t)NS;
  a.m.mode_a = q->scan->scan_processing ? 1u : 0u;
  if ((q->scan->flags & RPL_FLAG_PER_STREAM) != 0) a.m.lidars = cs->lidars;
  a.kept = w.kept;
  if (a.transform) {
    a.cloud_hdr = cs->xf_hdr;
    a.xf = cs->xf;
  }
  return a;
}

// on `st`, after the last push: the scan kernels or the cloud chain of every slot into w, then the tables
rpl_result msgs_prepare(rpl_capsule_stream* cs, rpl::MsgKind kind, const void* params, const MsgWork& w,
                        unsigned long long capacity, unsigned long long* offsets, uint32_t* sizes,
                        unsigned long long* total, cudaStream_t st) {
  rpl_ctx* c = cs->c;
  const size_t NS = (size_t)cs->n_streams * cs->max_scans, row = cs->max_nodes;
  rpl_result r = RPL_RESULT_OK;
  const rpl_scan_params* scan = msgs_scan_params(kind, params);
  for (uint32_t s0 = 0; s0 < cs->n_streams && r == RPL_RESULT_OK; s0 += cs->cloud_chunk) {
    const uint32_t ns = std::min(cs->cloud_chunk, cs->n_streams - s0);
    const size_t so = (size_t)s0 * cs->max_scans;
    if (scan) {
      const rpl_scan_params* p = scan;
      const rpl::ScanBatchArgs a = last_push_scans(cs, s0, ns);
      r = enqueue_scan(c, c->lane[0], reinterpret_cast<const rpl_node_hq*>(a.nodes), cs->scan_len + so, a.n_scans,
                       a.stride, p, nullptr, w.data + so * row, w.data + (NS + so) * row, w.counts + so, w.inc + so,
                       nullptr, nullptr, st, a.views, a.nodes_total,
                       lidar_table(cs, (p->flags & RPL_FLAG_PER_STREAM) != 0, s0));
      if (const rpl::ScanFilter* f = filters_at(cs, p, s0, ns); r == RPL_RESULT_OK && f)
        r = filter_scans(cs->c, f, footprints_at(cs, s0), cs->max_scans, a.n_scans, w.data + so * row,
                         w.data + (NS + so) * row, cs->max_nodes, nullptr, nullptr, w.counts + so, w.inc + so, st);
    } else {
      const auto* p = static_cast<const rpl_cloud_params*>(params);
      const rpl::ScanFootprint* fp = cloud_footprints_at(cs, p, s0, ns);
      r = stream_cloud_chunk(c, c->lane[0], last_push_scans(cs, s0, ns), lidars_at(cs, s0),
                             chains_at(cs, s0, fp != nullptr), cs->max_scans, p, w.data + so * row * 4, w.counts + so,
                             st, fp);
    }
  }
  if (r != RPL_RESULT_OK) return r;
  rpl::MsgTableArgs t{};
  if (kind == rpl::MsgKind::kScanCloud) {  // the kept counts size the messages
    const rpl::ScanCloudArgs a = scan_cloud_msg_args(cs, params, w);
    RPL_CUDA(c, rpl::launch_scan_cloud_count(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
    t.beams = w.counts;
    t.tail_bytes = a.transform ? a.tail_xf.bytes : a.tail.bytes;
    t.point_step = a.point_step;
  }
  if (kind == rpl::MsgKind::kRescan) t.bins = cs->rescan_bins;  // the LaserScans' beams and the entries size them
  t.kind = kind;
  t.hdr = (kind == rpl::MsgKind::kScanCloud || kind == rpl::MsgKind::kRescan) && scan_cloud_transforms(params)
              ? cs->xf_hdr
              : cs->msg_hdr;
  t.counts = kind == rpl::MsgKind::kScanCloud ? w.kept : w.counts;
  t.views = reinterpret_cast<const uint2*>(cs->views);
  t.n_slots = (uint32_t)NS;
  t.max_scans = cs->max_scans;
  t.capacity = capacity;
  t.offsets = offsets;
  t.sizes = sizes;
  t.total = total;
  if (kind == rpl::MsgKind::kPointCloud2 &&
      (static_cast<const rpl_cloud_params*>(params)->flags & RPL_CLOUD_PER_STREAM_CHAIN) != 0)
    t.clouds = cs->clouds;
  RPL_CUDA(c, rpl::launch_msg_table(t, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// the writers over slots [slot0, slot0 + n), message i at out + offsets[i] - out_base
rpl_result msgs_write(rpl_capsule_stream* cs, rpl::MsgKind kind, const void* params, long long clock_offset_ns,
                      const MsgWork& w, const unsigned long long* offsets, const uint32_t* sizes, uint32_t slot0,
                      uint32_t n, uint8_t* out, unsigned long long out_base, cudaStream_t st) {
  rpl_ctx* c = cs->c;
  if (n == 0) return RPL_RESULT_OK;
  const size_t NS = (size_t)cs->n_streams * cs->max_scans;
  rpl::MsgWriteArgs a{};
  a.hdr = cs->msg_hdr;
  if (cs->prev_stamped) {  // the stamps of the last push (an unstamped one kept none)
    a.begin_us = cs->slot_begin;
    a.end_us = cs->slot_end;
  }
  a.clock_offset_ns = clock_offset_ns;
  a.counts = w.counts;
  a.stride = cs->max_nodes;
  a.max_scans = cs->max_scans;
  a.slot0 = slot0;
  a.n = n;
  a.offsets = offsets;
  a.sizes = sizes;
  a.out = out;
  a.out_base = out_base;
  if (kind == rpl::MsgKind::kRescan) {  // the projection's LaserScans, transforms and window, with a's stamps and placement
    rpl::RescanArgs ra{};
    ra.c = scan_cloud_msg_args(cs, params, w);
    ra.c.m.slot0 = slot0;
    ra.c.m.n = n;
    ra.c.m.begin_us = a.begin_us;
    ra.c.m.clock_offset_ns = clock_offset_ns;
    ra.c.m.offsets = offsets;
    ra.c.m.sizes = sizes;
    ra.c.m.out = out;
    ra.c.m.out_base = out_base;
    ra.grid = cs->rescan;
    RPL_CUDA(c, rpl::launch_rescan(ra, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
    return RPL_RESULT_OK;
  }
  if (kind == rpl::MsgKind::kScanCloud) {  // the count pass's LaserScans and settings, with a's stamps and placement
    rpl::ScanCloudArgs sa = scan_cloud_msg_args(cs, params, w);
    sa.m.slot0 = slot0;
    sa.m.n = n;
    sa.m.begin_us = a.begin_us;
    sa.m.end_us = a.end_us;
    sa.m.clock_offset_ns = clock_offset_ns;
    sa.m.offsets = offsets;
    sa.m.sizes = sizes;
    sa.m.out = out;
    sa.m.out_base = out_base;
    RPL_CUDA(c, rpl::launch_scan_cloud(sa, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
    return RPL_RESULT_OK;
  }
  if (kind == rpl::MsgKind::kLaserScan) {
    a.ranges = w.data;
    a.intensities = w.data + NS * cs->max_nodes;
    a.angle_increment = w.inc;
    const auto* p = static_cast<const rpl_scan_params*>(params);
    a.mode_a = p->scan_processing ? 1u : 0u;
    if ((p->flags & RPL_FLAG_PER_STREAM) != 0) a.lidars = cs->lidars;
    RPL_CUDA(c, rpl::launch_laserscan_msgs(a, cs->max_nodes, st), RPL_RESULT_OPERATION_FAIL);
  } else {
    a.xyzi = w.data;
    static const rpl::CloudTail tail = cloud_tail();
    RPL_CUDA(c, rpl::launch_pointcloud2_msgs(a, tail, cs->max_nodes, st), RPL_RESULT_OPERATION_FAIL);
  }
  c->launches += (n + 65534) / 65535;
  return RPL_RESULT_OK;
}

rpl_result stream_msgs_dev(rpl_capsule_stream* cs, rpl::MsgKind kind, const void* params, int64_t clock_offset_ns,
                           uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                           uint64_t* total_bytes, void* stream) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  if (!stream_msgs_args_ok(cs, kind, params, msgs, msg_offsets, msg_sizes, total_bytes, true))
    return RPL_RESULT_INVALID_DATA;
  Carve k;
  msg_work_layout(cs, kind, false, k);
  return last_push_dev(cs, stream, k.bytes, [&](cudaStream_t st) -> rpl_result {
    Carve kw{cs->msg_work};
    const MsgWork w = msg_work_layout(cs, kind, false, kw);
    auto* offs = reinterpret_cast<unsigned long long*>(msg_offsets);
    rpl_result r = msgs_prepare(cs, kind, params, w, capacity, offs, msg_sizes,
                                reinterpret_cast<unsigned long long*>(total_bytes), st);
    if (r == RPL_RESULT_OK)
      r = msgs_write(cs, kind, params, clock_offset_ns, w, offs, msg_sizes, 0, cs->n_streams * cs->max_scans, msgs, 0,
                     st);
    return r;
  });
}

// a per-slot uint32 table of a packed call: the caller's host array and the device table behind it
struct SlotTable {
  uint32_t* host;
  const uint32_t* dev;
};

// The host form of a packed call (messages, nodes), once the caller has set the device and laid out its device tables:
// prepare(st) enqueues them on lane 0 behind the last push; the packed offsets, `tables` and the total are read back;
// when the total, in elements of elem bytes, fits capacity, each chunk of the last push -- one stretch [lo, hi) of the
// packed buffer -- is written by write(lane, s0, ns, lo) into the lane's stage and copied to out, followed by the
// chunk's slots of `rewritten` (nullable host), a table that write changes.
template <class Prepare, class Write>
rpl_result packed_host(rpl_capsule_stream* cs, Prepare prepare, uint64_t* offsets, const unsigned long long* offsets_dev,
                       std::initializer_list<SlotTable> tables, uint64_t* total, const unsigned long long* total_dev,
                       uint64_t capacity, const char* too_small, size_t elem, uint8_t* out, SlotTable rewritten,
                       Write write) {
  rpl_ctx* c = cs->c;
  const uint32_t NS = cs->n_streams * cs->max_scans;
  cudaStream_t st = c->lane[0].stream;
  for (int i = 0; i < kLanes; ++i) RPL_CUDA(c, cudaStreamWaitEvent(c->lane[i].stream, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
  if (const rpl_result r = prepare(st); r != RPL_RESULT_OK) {
    cudaStreamSynchronize(st);
    return r;
  }
  const cudaMemcpyKind d2h = cudaMemcpyDeviceToHost;
  RPL_CUDA(c, cudaMemcpyAsync(offsets, offsets_dev, (size_t)NS * 8, d2h, st), RPL_RESULT_OPERATION_FAIL);
  for (const SlotTable& t : tables)
    RPL_CUDA(c, cudaMemcpyAsync(t.host, t.dev, (size_t)NS * 4, d2h, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(total, total_dev, 8, d2h, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  const uint64_t end = *total;
  if (end > capacity) {
    c->err = too_small;
    return RPL_RESULT_INSUFFICIENT_MEMORY;
  }
  const uint32_t chunk = cs->cloud_chunk;
  auto stretch = [&](uint32_t s0, uint32_t ns) {
    const uint32_t i0 = s0 * cs->max_scans, i1 = (s0 + ns) * cs->max_scans;
    const uint64_t hi = i1 < NS ? std::min<uint64_t>(offsets[i1], end) : end;
    return std::make_pair(std::min<uint64_t>(offsets[i0], hi), hi);
  };
  size_t most = 0;
  for (uint32_t s0 = 0; s0 < cs->n_streams; s0 += chunk) {
    const auto [lo, hi] = stretch(s0, std::min(chunk, cs->n_streams - s0));
    most = std::max<size_t>(most, hi - lo);
  }
  if (const rpl_result g = grow_stage(c, kLanes, [&](Carve& k) { k.take<uint8_t>(most * elem); }); g != RPL_RESULT_OK)
    return g;
  auto run_chunk = [&](Lane& l, uint32_t s0, uint32_t ns) -> rpl_result {
    const auto [lo, hi] = stretch(s0, ns);
    if (hi == lo) return RPL_RESULT_OK;  // nothing of this chunk is packed: the tables read back stand
    RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);  // the lane's previous chunk has left
    const rpl_result r = write(l, s0, ns, lo);
    if (r != RPL_RESULT_OK) return r;
    RPL_CUDA(c, cudaMemcpyAsync(out + lo * elem, l.stage, (hi - lo) * elem, d2h, l.stream), RPL_RESULT_OPERATION_FAIL);
    if (rewritten.host) {
      const size_t so = (size_t)s0 * cs->max_scans;
      RPL_CUDA(c, cudaMemcpyAsync(rewritten.host + so, rewritten.dev + so, (size_t)ns * cs->max_scans * 4, d2h, l.stream),
               RPL_RESULT_OPERATION_FAIL);
    }
    return RPL_RESULT_OK;
  };
  return run_chunks(c, cs->n_streams, chunk, run_chunk);
}

rpl_result stream_msgs(rpl_capsule_stream* cs, rpl::MsgKind kind, const void* params, int64_t clock_offset_ns,
                       uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                       uint64_t* total_bytes) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!stream_msgs_args_ok(cs, kind, params, msgs, msg_offsets, msg_sizes, total_bytes, false))
    return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  Carve k;
  msg_work_layout(cs, kind, true, k);
  if (const rpl_result r = grow_msg_work(cs, k.bytes); r != RPL_RESULT_OK) return r;
  Carve kw{cs->msg_work};
  const MsgWork w = msg_work_layout(cs, kind, true, kw);
  return packed_host(
      cs, [&](cudaStream_t st) { return msgs_prepare(cs, kind, params, w, capacity, w.offsets, w.sizes, w.total, st); },
      msg_offsets, w.offsets, {{msg_sizes, w.sizes}}, total_bytes, w.total, capacity,
      "the messages need more than capacity bytes (total_bytes tells how many)", 1, msgs, SlotTable{},
      [&](Lane& l, uint32_t s0, uint32_t ns, uint64_t lo) {
        return msgs_write(cs, kind, params, clock_offset_ns, w, w.offsets, w.sizes, s0 * cs->max_scans,
                          ns * cs->max_scans, l.stage, lo, l.stream);
      });
}

// ---- messages from the push itself (DESIGN.md 5.7.1 "Messages from the push", "PointCloud2 messages from the push") --
// The push of in's kind, each chunk's scans written straight into their messages: per chunk, after the assembler, the
// directory places every slot behind the previous chunk's end; the scan kernels write each scan's arrays into its
// message; the header writer fills in the rest.  The device form writes into the caller's buffer and tables; the host
// form stages each chunk's messages on its lane and copies the stretch they fill.
// kind kPointCloud2 (params: rpl_cloud_params): per chunk, after the assembler, the cloud chain over the chunk's views
// into a block of one chunk's clouds (the device form: the session's message work block; the host form: the lane's),
// then the directory, which packs the messages exactly as msg_table_kernel does, then pointcloud2_msgs_kernel.  The
// push decodes and stamps with RPL_FLAG_PER_STREAM when the cloud takes RPL_CLOUD_PER_STREAM: of rpl_scan_params only
// that flag reaches the decoders, the assembler and the stamps.
// proj (kind kLaserScan, rpl_capsule_stream_push_scan_cloud_msgs*): each chunk also projects its LaserScan messages
// where they lie, into clouds (DESIGN.md 5.7.1 "LaserScans and their projected clouds from the push").
// The checks of a merge push that the set calls cannot make once for all: every group's members have equal enabled
// re-grid entries (pad aside) and equal re-grid headers under the push's cloud_params, and the merged outputs are there
bool merges_ok(rpl_capsule_stream* cs, const rpl_scan_cloud_params& proj, const rpl_msgs_out& merged, bool dev) {
  rpl_ctx* c = cs->c;
  if (!cs->mg_set) {
    c->err = "push_rescan_merge_msgs before the first rpl_capsule_stream_set_rescan_merges";
    return false;
  }
  if (!merged.msgs || !merged.msg_offsets || !merged.msg_sizes || !merged.total_bytes) {
    c->err = "null merged->msgs, msg_offsets, msg_sizes or total_bytes";
    return false;
  }
  if (dev && ((reinterpret_cast<uintptr_t>(merged.msgs) & 15u) || misaligned8(merged.msg_offsets) ||
              misaligned8(merged.total_bytes) || (reinterpret_cast<uintptr_t>(merged.msg_sizes) & 3u))) {
    c->err = "merged: msgs must be 16-byte aligned, msg_offsets and total_bytes 8-byte, msg_sizes 4-byte aligned";
    return false;
  }
  const std::vector<rpl::StreamMsgHeader>& hs =
      (proj.channels & rpl::kScanCloudPerStreamTransforms) ? cs->xf_hdr_host : cs->msg_hdr_host;
  for (uint32_t g = 0; g < cs->mg_groups; ++g) {
    const uint32_t b = cs->mg_begin_host[g], e = cs->mg_begin_host[g + 1];
    if (b == e) {
      c->err = "a merge group has no member";
      return false;
    }
    const uint32_t f = cs->mg_members_host[b];
    const rpl_rescan_settings& t0 = cs->rescan_host[f];
    const rpl::StreamMsgHeader& h0 = hs[f];
    for (uint32_t j = b; j < e; ++j) {
      const uint32_t s = cs->mg_members_host[j];
      if (!cs->rescan_host[s].enabled || std::memcmp(&cs->rescan_host[s], &t0, offsetof(rpl_rescan_settings, pad))) {
        c->err = "a merge group's members need equal enabled rpl_rescan_settings entries";
        return false;
      }
      if (hs[s].bytes != h0.bytes || std::memcmp(hs[s].w, h0.w, h0.bytes)) {
        c->err = "a merge group's re-grid messages need one frame_id";
        return false;
      }
    }
  }
  return true;
}

rpl_result push_msgs(rpl_capsule_stream* cs, const rpl_push_input* in, rpl::MsgKind kind, const void* params,
                     int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                     uint64_t* total_bytes, uint32_t* scans_per_stream, bool dev, void* stream,
                     const rpl_scan_cloud_params* proj = nullptr, const rpl_msgs_out* clouds = nullptr,
                     bool rescan = false, const rpl_msgs_out* merged = nullptr) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  cs->cloud_chunk = 0;  // as a push that fails its checks
  if (!in || !params || !msgs || !msg_offsets || !msg_sizes || !total_bytes || !scans_per_stream) {
    c->err = "null input, params, msgs, msg_offsets, msg_sizes, total_bytes or scans_per_stream";
    return RPL_RESULT_INVALID_DATA;
  }
  if (proj) {
    if (!clouds->msgs || !clouds->msg_offsets || !clouds->msg_sizes || !clouds->total_bytes) {
      c->err = "null clouds->msgs, msg_offsets, msg_sizes or total_bytes";
      return RPL_RESULT_INVALID_DATA;
    }
    if (!scan_cloud_call_ok(cs, *proj)) return RPL_RESULT_INVALID_DATA;
    if (rescan && cs->rescan_host.empty()) {
      c->err = "push_rescan_msgs before the first rpl_capsule_stream_set_rescans";
      return RPL_RESULT_INVALID_DATA;
    }
    if (merged && !merges_ok(cs, *proj, *merged, dev)) return RPL_RESULT_INVALID_DATA;
    if (dev && ((reinterpret_cast<uintptr_t>(clouds->msgs) & 15u) || misaligned8(clouds->msg_offsets) ||
                misaligned8(clouds->total_bytes) || (reinterpret_cast<uintptr_t>(clouds->msg_sizes) & 3u))) {
      c->err = "clouds: msgs must be 16-byte aligned, msg_offsets and total_bytes 8-byte, msg_sizes 4-byte aligned";
      return RPL_RESULT_INVALID_DATA;
    }
  }
  if (in->chunk_bytes != 0 && (!cs->bytes || !in->rx_us)) {
    c->err = cs->bytes ? "chunk_bytes is a stamped push's (rx_us set)"
                       : "chunk_bytes is a byte push's: a framed session's receive times are per capsule";
    return RPL_RESULT_INVALID_DATA;
  }
  auto mis4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) != 0; };
  if (dev && ((reinterpret_cast<uintptr_t>(msgs) & 15u) || misaligned8(msg_offsets) || misaligned8(total_bytes) ||
              mis4(msg_sizes) || mis4(scans_per_stream))) {
    c->err = "msgs must be 16-byte aligned, msg_offsets and total_bytes 8-byte, msg_sizes and scans_per_stream 4-byte "
             "aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  const bool cloud = kind == rpl::MsgKind::kPointCloud2;
  const auto* cp = cloud ? static_cast<const rpl_cloud_params*>(params) : nullptr;
  if (cloud && !cloud_call_ok(cs, cp)) return RPL_RESULT_INVALID_DATA;
  // a cloud push's: its decode, assemble and stamp settings (RPL_CLOUD_PER_STREAM before set_lidars fails the push's
  // check of RPL_FLAG_PER_STREAM)
  rpl_scan_params push_params{};
  if (cloud && (cp->flags & RPL_CLOUD_PER_STREAM) != 0) push_params.flags = RPL_FLAG_PER_STREAM;
  const auto* sp_params = cloud ? &push_params : static_cast<const rpl_scan_params*>(params);
  if (!cs->push_msg_work) {  // the first message push: the session's tables, made once (their size is fixed)
    RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
    Carve k;
    push_msg_work_layout(cs, k);
    RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&cs->push_msg_work), k.bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
    RPL_CUDA(c, cudaMallocHost(reinterpret_cast<void**>(&cs->push_msg_extent), kLanes * 3 * 8),
             RPL_RESULT_INSUFFICIENT_MEMORY);
    for (cudaEvent_t& e : cs->push_msg_extent_ready)
      RPL_CUDA(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaEventCreateWithFlags(&cs->push_msg_dir_order, cudaEventDisableTiming), RPL_RESULT_OPERATION_FAIL);
  }
  // the first projecting or re-gridding push: its tables, made once (a re-gridding push uses the carry alone)
  if (proj && !cs->push_scan_cloud_work) {
    RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
    Carve k;
    scan_cloud_work_layout(cs, k);
    RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&cs->push_scan_cloud_work), k.bytes),
             RPL_RESULT_INSUFFICIENT_MEMORY);
    RPL_CUDA(c, cudaMallocHost(reinterpret_cast<void**>(&cs->push_scan_cloud_extent), kLanes * 3 * 8),
             RPL_RESULT_INSUFFICIENT_MEMORY);
    RPL_CUDA(c, cudaEventCreateWithFlags(&cs->push_scan_cloud_dir_order, cudaEventDisableTiming),
             RPL_RESULT_OPERATION_FAIL);
  }
  Carve k{cs->push_msg_work};
  PushMsgs pm{msgs, capacity, msg_offsets, msg_sizes, total_bytes, clock_offset_ns, push_msg_work_layout(cs, k), cp,
              nullptr, nullptr};
  if (proj) {
    Carve kp{cs->push_scan_cloud_work};
    const ScanCloudWork sw = scan_cloud_work_layout(cs, kp);
    pm.proj = proj;
    pm.clouds = clouds;
    pm.proj_carry = sw.carry;
    pm.kept = sw.kept;
    pm.rescan = rescan;
    if (proj->channels & rpl::kScanCloudPerStreamTransforms) {
      pm.proj_hdr = cs->xf_hdr;
      pm.proj_xf = cs->xf;
    }
  }
  if (merged && !dev) {  // the host form's staging: the groups' directory and their messages' bound
    uint32_t hdr_most = 0, bins_most = 0;  // a held grid's message may have taken either header
    for (uint32_t s : cs->mg_streams_host) {
      hdr_most = std::max(hdr_most, cs->msg_hdr_host[s].bytes);
      if (!cs->xf_hdr_host.empty()) hdr_most = std::max(hdr_most, cs->xf_hdr_host[s].bytes);
      bins_most = std::max(bins_most, rescan_bins(cs->rescan_host[s]));
    }
    Carve kd;
    merge_stage_layout(kd, cs->mg_groups);
    const size_t bytes = kd.bytes + (size_t)cs->mg_groups * ((hdr_most + 36 + 4 * (size_t)bins_most + 15) & ~(size_t)15);
    if (bytes > cs->mg_stage_bytes) {
      RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
      unsigned char* b = nullptr;
      RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&b), bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
      cudaFree(cs->mg_stage);  // its last user, a host push, has synchronised
      cs->mg_stage = b;
      cs->mg_stage_bytes = bytes;
    }
  }
  pm.merged = merged;
  if (cloud && dev) {  // one chunk's clouds, in the session's message work block (cloud_msgs' when that is larger)
    const size_t NS = (size_t)cs->chunk_dev * cs->max_scans;
    auto layout = [&](Carve& kw) {
      pm.xyzi = kw.take<float>(NS * cs->max_nodes * 4);
      pm.points = kw.take<uint32_t>(NS);
    };
    Carve kb;
    layout(kb);
    RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
    if (const rpl_result r = grow_msg_work(cs, kb.bytes); r != RPL_RESULT_OK) return r;
    Carve kw{cs->msg_work};
    layout(kw);
  }
  StampPush sp{};
  const bool stamped = in->rx_us != nullptr;
  // (a stamped push's scan stamps stay on the device: the messages carry them)
  if (stamped && !stamp_args_ok(cs, sp_params, in->timing, in->rx_us, cs->bytes ? in->chunk_bytes : 1u,
                                reinterpret_cast<uint64_t*>(pm.w.ts), &sp))
    return RPL_RESULT_INVALID_DATA;
  const uint32_t sample_duration_us = stamped ? (in->timing ? in->timing->sample_duration_us : 0u) : in->sample_duration_us;
  const rpl_result r = stream_push(cs, in->data, in->counts, sample_duration_us, sp_params, nullptr, nullptr, nullptr,
                                   nullptr, scans_per_stream, stamped ? &sp : nullptr, cs->bytes, dev, stream, &pm);
  if (r != RPL_RESULT_OK) return r;
  if (merged) cs->mg_seq++;
  if (!dev && (*total_bytes > capacity || (proj && *clouds->total_bytes > clouds->capacity) ||
               (merged && *merged->total_bytes > merged->capacity))) {  // windows and held grids advanced
    c->err = "the messages need more than capacity bytes (total_bytes tells how many; the push itself is done)";
    return RPL_RESULT_INSUFFICIENT_MEMORY;
  }
  return RPL_RESULT_OK;
}

// rescan: rpl_capsule_stream_push_rescan_msgs*, whose `clouds` are the re-grid messages; merge: a merge push
// (rpl_capsule_stream_push_rescan_merge_msgs*), whose merged scans go into `merged`
rpl_result push_scan_cloud_msgs(rpl_capsule_stream* cs, const rpl_push_input* in, const rpl_scan_params* scan_params,
                                const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                const rpl_msgs_out* scans, const rpl_msgs_out* clouds, uint32_t* scans_per_stream,
                                bool dev, void* stream, bool rescan = false, bool merge = false,
                                const rpl_msgs_out* merged = nullptr) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  if (!scans || !clouds || !cloud_params || (merge && !merged)) {
    cs->cloud_chunk = 0;  // as a push that fails its checks
    cs->c->err = merge    ? "null scans, rescans, merged or cloud_params"
                 : rescan ? "null scans, rescans or cloud_params"
                          : "null scans, clouds or cloud_params";
    return RPL_RESULT_INVALID_DATA;
  }
  return push_msgs(cs, in, rpl::MsgKind::kLaserScan, scan_params, clock_offset_ns, scans->msgs, scans->capacity,
                   scans->msg_offsets, scans->msg_sizes, scans->total_bytes, scans_per_stream, dev, stream,
                   cloud_params, clouds, rescan, merged);
}

// ---- grabbed node buffers of the last push (DESIGN.md 5.7.1 "Session nodes") -------------------------------------
// Per call: the directory over every slot (counts, packed offsets, each slot's place), then per chunk of the push the
// shared-memory EMIT kernel with the general kernel behind it for the ascended slots, writing each revolution at its
// place, and the gather for the others.  The device form places into the caller's buffer; the host form reads the
// directory back first and then places and copies chunk by chunk over the lanes, each chunk's buffers being one
// stretch of the packed buffer, so that only node bytes cross the link.

bool stream_nodes_args_ok(rpl_capsule_stream* cs, const void* nodes, const void* offsets, const void* counts,
                          const void* status, const void* total, bool dev) {
  rpl_ctx* c = cs->c;
  if (!nodes || !offsets || !counts || !status || !total) {
    c->err = "null nodes, node_offsets, node_counts, status or total_nodes";
    return false;
  }
  auto mis4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) != 0; };
  if (dev && ((reinterpret_cast<uintptr_t>(nodes) & 15u) || misaligned8(offsets) || misaligned8(total) || mis4(counts) ||
              mis4(status))) {
    c->err = "nodes must be 16-byte aligned, node_offsets and total_nodes 8-byte, node_counts and status 4-byte aligned";
    return false;
  }
  if (cs->cloud_chunk == 0) {
    c->err = "no nodes to take: the session has not pushed yet, or its last push failed";
    return false;
  }
  return true;
}

// which kernels a nodes call needs: the scan kernels (some stream is ascended), the gather (some stream is not)
struct NodeKinds {
  bool ascended, passed;
};
NodeKinds node_kinds(const rpl_capsule_stream* cs, uint32_t apply_ascend, const uint8_t* per_stream) {
  if (!per_stream) return NodeKinds{apply_ascend != 0, apply_ascend == 0};
  NodeKinds k{false, false};
  for (uint32_t s = 0; s < cs->n_streams; ++s) (per_stream[s] ? k.ascended : k.passed) = true;
  return k;
}

// on `st`, after the last push: the per-stream flags to the device, then the directory of every slot
rpl_result nodes_prepare(rpl_capsule_stream* cs, const NodeWork& w, uint32_t apply_ascend, const uint8_t* per_stream,
                         unsigned long long capacity, unsigned long long* offsets, uint32_t* counts, uint32_t* status,
                         unsigned long long* total, bool rebase, cudaStream_t st) {
  rpl_ctx* c = cs->c;
  if (per_stream)
    RPL_CUDA(c, cudaMemcpyAsync(w.ascend, per_stream, cs->n_streams, cudaMemcpyHostToDevice, st), RPL_RESULT_OPERATION_FAIL);
  rpl::NodeDirArgs a{};
  a.views = reinterpret_cast<const uint2*>(cs->views);
  a.n_slots = cs->n_streams * cs->max_scans;
  a.max_scans = cs->max_scans;
  a.chunk_slots = cs->cloud_chunk * cs->max_scans;
  a.rebase = rebase ? 1u : 0u;
  a.ascend = per_stream ? w.ascend : nullptr;
  a.ascend_all = apply_ascend;
  a.capacity = capacity;
  a.offsets = offsets;
  a.counts = counts;
  a.status = status;
  a.total = total;
  a.place = w.place;
  RPL_CUDA(c, rpl::launch_node_directory(a, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// The buffers of the scans of one chunk of the last push (last_push_scans), placed behind `out`; status points at the
// chunk's first slot.  One EMIT instantiation
// serves every ascended slot: the ascended buffer does not depend on the LaserScan mode, and no LaserScan is computed.
rpl_result stream_nodes_chunk(rpl_capsule_stream* cs, Lane& l, uint32_t s0, uint32_t ns, NodeKinds kinds,
                              const unsigned long long* place, rpl_node_hq* out, uint32_t* status, cudaStream_t st) {
  rpl_ctx* c = cs->c;
  rpl::ScanBatchArgs a = last_push_scans(cs, s0, ns);
  a.nodes_out = reinterpret_cast<uint2*>(out);
  a.out_first = place + (size_t)s0 * cs->max_scans;
  a.status = status;
  a.apply_ascend = 1;
  a.fallback_list = l.fallback_list;
  if (kinds.ascended) {
    rpl_result r = scratch_enter(c, l, st);
    if (r == RPL_RESULT_OK) r = enqueue_args(c, l, a, 0u, st);
    if (r == RPL_RESULT_OK) r = scratch_leave(c, l, st);
    if (r != RPL_RESULT_OK) return r;
  }
  if (kinds.passed) {
    const rpl::NodeGatherArgs g{a.nodes, a.views, a.out_first, a.n_scans, a.nodes_out};
    RPL_CUDA(c, rpl::launch_node_gather(g, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
    c->launches++;
  }
  return RPL_RESULT_OK;
}

rpl_result stream_nodes_dev(rpl_capsule_stream* cs, uint32_t apply_ascend, const uint8_t* per_stream, rpl_node_hq* nodes,
                            uint64_t capacity, uint64_t* node_offsets, uint32_t* node_counts, uint32_t* status,
                            uint64_t* total_nodes, void* stream) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  if (!stream_nodes_args_ok(cs, nodes, node_offsets, node_counts, status, total_nodes, true)) return RPL_RESULT_INVALID_DATA;
  Carve k{cs->node_work};
  const NodeWork w = node_work_layout(cs, k);
  // (an earlier nodes call reads the same tables: behind the last push, it is done before these too)
  return last_push_dev(cs, stream, 0, [&](cudaStream_t st) -> rpl_result {
    rpl_result r = nodes_prepare(cs, w, apply_ascend, per_stream, capacity,
                                 reinterpret_cast<unsigned long long*>(node_offsets), node_counts, status,
                                 reinterpret_cast<unsigned long long*>(total_nodes), false, st);
    const NodeKinds kinds = node_kinds(cs, apply_ascend, per_stream);
    for (uint32_t s0 = 0; s0 < cs->n_streams && r == RPL_RESULT_OK; s0 += cs->cloud_chunk)
      r = stream_nodes_chunk(cs, cs->c->lane[0], s0, std::min(cs->cloud_chunk, cs->n_streams - s0), kinds, w.place,
                             nodes, status + (size_t)s0 * cs->max_scans, st);
    return r;
  });
}

rpl_result stream_nodes(rpl_capsule_stream* cs, uint32_t apply_ascend, const uint8_t* per_stream, rpl_node_hq* nodes,
                        uint64_t capacity, uint64_t* node_offsets, uint32_t* node_counts, uint32_t* status,
                        uint64_t* total_nodes) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (!stream_nodes_args_ok(cs, nodes, node_offsets, node_counts, status, total_nodes, false)) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  Carve k{cs->node_work};
  const NodeWork w = node_work_layout(cs, k);
  const NodeKinds kinds = node_kinds(cs, apply_ascend, per_stream);
  // an ascended chunk's kernels rewrite its statuses
  return packed_host(
      cs,
      [&](cudaStream_t st) {
        return nodes_prepare(cs, w, apply_ascend, per_stream, capacity, w.offsets, w.counts, w.status, w.total, true, st);
      },
      node_offsets, w.offsets, {{node_counts, w.counts}, {status, w.status}}, total_nodes, w.total, capacity,
      "the buffers need more than capacity_nodes nodes (total_nodes tells how many)", sizeof(rpl_node_hq),
      reinterpret_cast<uint8_t*>(nodes), SlotTable{kinds.ascended ? status : nullptr, w.status},
      [&](Lane& l, uint32_t s0, uint32_t ns, uint64_t) {
        return stream_nodes_chunk(cs, l, s0, ns, kinds, w.place, reinterpret_cast<rpl_node_hq*>(l.stage),
                                  w.status + (size_t)s0 * cs->max_scans, l.stream);
      });
}

}  // namespace

extern "C" {

// ---- wire bytes -> LaserScan in one host call: a fresh dense session's host push, with nothing kept ----------------
rpl_result rpl_chain_dense_laserscan(rpl_ctx* c, const uint8_t* capsules, const uint32_t* capsule_counts,
                                     uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                     const rpl_scan_params* params, uint32_t max_nodes, uint32_t max_scans,
                                     float* ranges, float* intensities, uint32_t* beam_counts, float* angle_increment,
                                     uint32_t* scans_per_stream) {
  if (!c || !capsules || !capsule_counts || !params || !ranges || !intensities || !beam_counts || !scans_per_stream)
    return RPL_RESULT_INVALID_DATA;
  if (n_streams == 0) return RPL_RESULT_OK;
  if (max_nodes == 0 || max_nodes > rpl::kSmallMaxNodes || (max_nodes & 1u) || max_scans == 0 || stride_capsules == 0) {
    c->err = "need an even max_nodes in [2, 8192] (the longest revolution), max_scans > 0, stride_capsules > 0";
    return RPL_RESULT_INVALID_DATA;
  }
  for (uint32_t s = 0; s < n_streams; ++s)
    if (capsule_counts[s] > stride_capsules) {
      c->err = "capsule_counts[s] exceeds stride_capsules";
      return RPL_RESULT_INVALID_DATA;
    }
  // chunk: about 16 MiB of capsules (~64 MiB of decoded nodes), whole streams
  const size_t cap_bytes_stream = (size_t)stride_capsules * 84;
  uint32_t chunk = (uint32_t)std::max<size_t>(1, ((size_t)16 << 20) / cap_bytes_stream);
  chunk = std::min(chunk, n_streams);
  if ((size_t)chunk * max_scans > c->max_scans) chunk = c->max_scans / max_scans;
  if (chunk == 0) {
    c->err = "the context's max_scans is smaller than max_scans of one stream";
    return RPL_RESULT_INVALID_DATA;
  }
  const size_t nodes_stream = (size_t)stride_capsules * 40;
  if ((size_t)chunk * nodes_stream > 0xFFFFFFFFull) {
    c->err = "chunk too large for 32-bit views";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!sample_duration_ok(c, sample_duration_us)) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  // a chunk's decoded nodes, reports, scan-start lists and views sit in the lane block behind its input and outputs
  auto chunk_at = [&](Carve& k, uint32_t) {
    WireChunk w{};
    w.ans_type = 0x85;
    w.stride_capsules = stride_capsules;
    w.max_nodes = max_nodes;
    w.max_scans = max_scans;
    w.stride_nodes = (uint32_t)nodes_stream;
    w.starts_stride = 2 * max_scans + 64;  // scan starts per stream the decoder may list
    w.nodes = k.take<rpl_node_hq>(chunk * nodes_stream);
    w.node_counts = k.take<uint32_t>(chunk);
    w.status = k.take<uint32_t>((size_t)chunk * stride_capsules);
    w.offsets = k.take<uint32_t>((size_t)chunk * stride_capsules);
    w.starts = k.take<uint32_t>((size_t)chunk * w.starts_stride);
    w.start_counts = k.take<uint32_t>(chunk);
    w.views = k.take<rpl_scan_view>((size_t)chunk * max_scans);
    w.scan_len = k.take<uint32_t>((size_t)chunk * max_scans);
    return w;
  };
  const HostWire h{capsules, capsule_counts, cap_bytes_stream, sample_duration_us, max_nodes, max_scans, params, ranges,
                   intensities, angle_increment, beam_counts, scans_per_stream, nullptr, 0};
  return push_host(c, h, n_streams, chunk, chunk_at);
}

rpl_result rpl_capsule_stream_create(rpl_ctx* c, uint32_t ans_type, uint32_t n_streams, uint32_t stride_capsules,
                                     uint32_t max_nodes, uint32_t max_scans, rpl_capsule_stream** out) {
  if (!c || !out) return RPL_RESULT_INVALID_DATA;
  *out = nullptr;
  if (rpl_capsule_bytes(ans_type) == 0) {
    c->err = "a stream session takes the capsule answer types 0x82..0x86 (0x81 standard-node bytes: "
             "rpl_capsule_stream_create_bytes)";
    return RPL_RESULT_INVALID_DATA;
  }
  return stream_create(c, ans_type, false, n_streams, stride_capsules, max_nodes, max_scans, out);
}

void rpl_capsule_stream_destroy(rpl_capsule_stream* cs) {
  if (!cs) return;
  cudaSetDevice(cs->c->device);
  if (cs->done) cudaEventSynchronize(cs->done);
  for (int i = 0; i < kLanes; ++i) cudaStreamSynchronize(cs->c->lane[i].stream);
  for (int p = 0; p < 2; ++p) {
    cudaFree(cs->arena[p]);
    cudaFree(cs->carry_len[p]);
    cudaFree(cs->open_ts[p]);
  }
  cudaFree(cs->held_rx);
  cudaFree(cs->scan_ends);
  cudaFree(cs->held);
  cudaFree(cs->status);
  cudaFree(cs->offsets);
  cudaFree(cs->node_counts);
  cudaFree(cs->starts);
  cudaFree(cs->start_counts);
  cudaFree(cs->scan_len);
  cudaFree(cs->views);
  cudaFree(cs->framer);
  cudaFree(cs->framed);
  cudaFree(cs->framed_counts);
  cudaFree(cs->framed_rx);
  cudaFree(cs->lists[0]);
  cudaFree(cs->lists[1]);
  cudaFree(cs->slot_begin);
  cudaFree(cs->slot_end);
  cudaFree(cs->msg_hdr);
  cudaFree(cs->msg_work);
  cudaFree(cs->node_work);
  cudaFree(cs->lidars);
  cudaFree(cs->clouds);
  cudaFree(cs->clouds_fp);
  cudaFree(cs->filters);
  cudaFree(cs->footprints);
  cudaFree(cs->counters);
  cudaFree(cs->push_msg_work);
  cudaFree(cs->migrate_work);
  cudaFreeHost(cs->push_msg_extent);
  for (cudaEvent_t e : cs->push_msg_extent_ready)
    if (e) cudaEventDestroy(e);
  if (cs->push_msg_dir_order) cudaEventDestroy(cs->push_msg_dir_order);
  cudaFree(cs->push_scan_cloud_work);
  cudaFree(cs->xf);
  cudaFree(cs->xf_hdr);
  cudaFree(cs->rescan);
  cudaFree(cs->rescan_bins);
  cudaFree(cs->win);
  cudaFree(cs->win_state);
  cudaFree(cs->win_ring);
  cudaFree(cs->win_streams);
  cudaFree(cs->mg_block);
  cudaFree(cs->mg_stage);
  cudaFreeHost(cs->push_scan_cloud_extent);
  if (cs->push_scan_cloud_dir_order) cudaEventDestroy(cs->push_scan_cloud_dir_order);
  if (cs->done) cudaEventDestroy(cs->done);
  delete cs;
}

rpl_result rpl_capsule_stream_push(rpl_capsule_stream* cs, const uint8_t* capsules, const uint32_t* capsule_counts,
                                   uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                   float* intensities, uint32_t* beam_counts, float* angle_increment,
                                   uint32_t* scans_per_stream) {
  return stream_push(cs, capsules, capsule_counts, sample_duration_us, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, nullptr, false, false, nullptr);
}

rpl_result rpl_capsule_stream_push_dev(rpl_capsule_stream* cs, const uint8_t* capsules, const uint32_t* capsule_counts,
                                       uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                       float* intensities, uint32_t* beam_counts, float* angle_increment,
                                       uint32_t* scans_per_stream, void* stream) {
  return stream_push(cs, capsules, capsule_counts, sample_duration_us, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, nullptr, false, true, stream);
}

rpl_result rpl_capsule_stream_push_ts(rpl_capsule_stream* cs, const uint8_t* capsules, const uint32_t* capsule_counts,
                                      const rpl_timing* timing, const uint64_t* capsule_rx_us,
                                      const rpl_scan_params* params, float* ranges, float* intensities,
                                      uint32_t* beam_counts, float* angle_increment, uint32_t* scans_per_stream,
                                      uint64_t* scan_begin_ts_us) {
  StampPush sp{};
  if (!stamp_args_ok(cs, params, timing, capsule_rx_us, 1, scan_begin_ts_us, &sp)) return RPL_RESULT_INVALID_DATA;
  return stream_push(cs, capsules, capsule_counts, timing ? timing->sample_duration_us : 0u, params, ranges, intensities,
                     beam_counts, angle_increment, scans_per_stream, &sp, false, false, nullptr);
}

rpl_result rpl_capsule_stream_push_ts_dev(rpl_capsule_stream* cs, const uint8_t* capsules,
                                          const uint32_t* capsule_counts, const rpl_timing* timing,
                                          const uint64_t* capsule_rx_us, const rpl_scan_params* params, float* ranges,
                                          float* intensities, uint32_t* beam_counts, float* angle_increment,
                                          uint32_t* scans_per_stream, uint64_t* scan_begin_ts_us, void* stream) {
  StampPush sp{};
  if (!stamp_args_ok(cs, params, timing, capsule_rx_us, 1, scan_begin_ts_us, &sp)) return RPL_RESULT_INVALID_DATA;
  return stream_push(cs, capsules, capsule_counts, timing ? timing->sample_duration_us : 0u, params, ranges, intensities,
                     beam_counts, angle_increment, scans_per_stream, &sp, false, true, stream);
}

rpl_result rpl_capsule_stream_reset(rpl_capsule_stream* cs, const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  cudaStream_t st = c->lane[0].stream;
  RPL_CUDA(c, cudaStreamWaitEvent(st, cs->done, 0), RPL_RESULT_OPERATION_FAIL);
  const uint32_t p = cs->parity;
  for (uint32_t s = 0; s < cs->n_streams;) {  // one pair of clears per run of masked streams
    if (stream_mask && !stream_mask[s]) {
      ++s;
      continue;
    }
    uint32_t e = s + 1;
    while (e < cs->n_streams && (!stream_mask || stream_mask[e])) ++e;
    RPL_CUDA(c, cudaMemsetAsync(cs->held + (size_t)s * rpl::kHeldWords, 0, (size_t)(e - s) * rpl::kHeldWords * 4, st),
             RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemsetAsync(cs->carry_len[p] + s, 0, (size_t)(e - s) * 4, st), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemsetAsync(cs->open_ts[p] + s, 0, (size_t)(e - s) * 8, st), RPL_RESULT_OPERATION_FAIL);
    RPL_CUDA(c, cudaMemsetAsync(cs->held_rx + s, 0, (size_t)(e - s) * 8, st), RPL_RESULT_OPERATION_FAIL);
    if (cs->framer)  // the handlers' reset: _cached_scan_node_buf_pos = 0, _is_previous_capsuledataRdy = false
      RPL_CUDA(c, cudaMemsetAsync(cs->framer + (size_t)s * rpl::kFramerWords, 0, (size_t)(e - s) * rpl::kFramerWords * 4, st),
               RPL_RESULT_OPERATION_FAIL);
    if (cs->win_state)  // the windows over the re-gridded scans start over
      RPL_CUDA(c, cudaMemsetAsync(cs->win_state + s, 0, (size_t)(e - s) * sizeof(uint2), st), RPL_RESULT_OPERATION_FAIL);
    s = e;
  }
  if (const rpl_result r = merges_empty(cs, stream_mask, st); r != RPL_RESULT_OK) return r;  // and the held grids
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_capsule_stream_state(rpl_capsule_stream* cs, uint32_t* open_nodes, uint32_t* held_capsule,
                                    uint32_t* held_bytes) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);
  if (open_nodes)
    RPL_CUDA(c, cudaMemcpy(open_nodes, cs->carry_len[cs->parity], (size_t)cs->n_streams * 4, cudaMemcpyDeviceToHost),
             RPL_RESULT_OPERATION_FAIL);
  std::vector<uint32_t> fr;  // a capsule byte session's framer records
  if (cs->framer && (held_capsule || held_bytes)) {
    fr.resize((size_t)cs->n_streams * rpl::kFramerWords);
    RPL_CUDA(c, cudaMemcpy(fr.data(), cs->framer, fr.size() * 4, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  }
  // the held records: HQ's stays zero; 0x81's holds the byte machine's state, 0..4 bytes held
  std::vector<uint32_t> h;
  if (held_capsule || held_bytes) {
    h.resize((size_t)cs->n_streams * rpl::kHeldWords);
    RPL_CUDA(c, cudaMemcpy(h.data(), cs->held, h.size() * 4, cudaMemcpyDeviceToHost), RPL_RESULT_OPERATION_FAIL);
  }
  for (uint32_t s = 0; s < cs->n_streams; ++s) {
    const bool normal = (cs->types.empty() ? cs->ans_type : cs->types[s]) == RPL_ANS_MEASUREMENT;
    const uint32_t ok = h.empty() ? 0u : h[(size_t)s * rpl::kHeldWords + rpl::kHeldOk];
    const uint32_t* f = fr.empty() || normal ? nullptr : fr.data() + (size_t)s * rpl::kFramerWords;
    // skipped bytes waiting to be reported: the next frame releases nothing (the SDK cleared its ready flag)
    if (held_capsule) held_capsule[s] = normal || (f && f[rpl::kFramerLost]) ? 0u : ok;
    if (held_bytes) held_bytes[s] = normal ? ok : f ? f[rpl::kFramerPos] : 0u;
  }
  return RPL_RESULT_OK;
}

rpl_result rpl_capsule_stream_counters(rpl_capsule_stream* cs, rpl_stream_counters* out, const uint8_t* clear_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // host pushes return synchronised
  if (out)
    RPL_CUDA(c, cudaMemcpy(out, cs->counters, (size_t)cs->n_streams * sizeof(rpl_stream_counters), cudaMemcpyDeviceToHost),
             RPL_RESULT_OPERATION_FAIL);
  if (!clear_mask) return RPL_RESULT_OK;
  cudaStream_t st = c->lane[0].stream;
  for (uint32_t s = 0; s < cs->n_streams;) {  // one clear per run of masked streams
    if (!clear_mask[s]) {
      ++s;
      continue;
    }
    uint32_t e = s + 1;
    while (e < cs->n_streams && clear_mask[e]) ++e;
    RPL_CUDA(c, cudaMemsetAsync(cs->counters + s, 0, (size_t)(e - s) * sizeof(rpl::StreamCounters), st),
             RPL_RESULT_OPERATION_FAIL);
    s = e;
  }
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);  // cleared before any later push runs
  return RPL_RESULT_OK;
}

// ---- moving streams between sessions (DESIGN.md 5.7.1): records of each stream's carried state ----
}  // extern "C"

namespace {

static_assert(rpl::kRecVersion == RPL_STREAM_RECORD_VERSION && rpl::kRecCounterBytes == sizeof(rpl_stream_counters),
              "the record of include/rpl_b200.h");

// a record's bytes, rounded up to 16: its fixed part (with the framer record for a capsule answer type in a byte
// session) and L nodes
uint64_t record_bytes(bool bytes, uint32_t ans_type, uint32_t L) {
  return ((uint64_t)rpl::record_fixed_bytes(bytes && ans_type != RPL_ANS_MEASUREMENT) + 8ull * L + 15ull) & ~15ull;
}

uint32_t stream_type(const rpl_capsule_stream* cs, uint32_t s) { return cs->types.empty() ? cs->ans_type : cs->types[s]; }

// The device staging of n records, `bytes` in all, then their tables: offsets [n], streams [n], types [n] (uploaded as
// one block from `tables`), in args a.  No device call of the session may be in flight.
rpl_result migrate_stage(rpl_capsule_stream* cs, uint64_t bytes, uint32_t n, const std::vector<unsigned char>& tables,
                         rpl::MigrateArgs* a) {
  rpl_ctx* c = cs->c;
  const size_t rec = (size_t)((bytes + 15) & ~15ull), need = rec + tables.size();
  if (cs->migrate_work_bytes < need) {
    cudaFree(cs->migrate_work);
    cs->migrate_work = nullptr;
    cs->migrate_work_bytes = 0;
    RPL_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&cs->migrate_work), need), RPL_RESULT_INSUFFICIENT_MEMORY);
    cs->migrate_work_bytes = need;
  }
  RPL_CUDA(c, cudaMemcpyAsync(cs->migrate_work + rec, tables.data(), tables.size(), cudaMemcpyHostToDevice,
                              c->lane[0].stream),
           RPL_RESULT_OPERATION_FAIL);
  const uint32_t p = cs->parity;
  a->records = cs->migrate_work;
  a->offsets = reinterpret_cast<const unsigned long long*>(cs->migrate_work + rec);
  a->streams = reinterpret_cast<const uint32_t*>(cs->migrate_work + rec + (size_t)8 * n);
  a->types = reinterpret_cast<const uint32_t*>(cs->migrate_work + rec + (size_t)12 * n);
  a->n = n;
  a->arena = reinterpret_cast<uint2*>(cs->arena[p]);
  a->stride_nodes = cs->stride_nodes;
  a->max_nodes = cs->max_nodes;
  a->carry_len = cs->carry_len[p];
  a->open_ts = cs->open_ts[p];
  a->held_rx = cs->held_rx;
  a->held = cs->held;
  a->framer = cs->framer;
  a->counters = cs->counters;
  a->kind = cs->bytes ? 1u : 0u;
  return RPL_RESULT_OK;
}

// the tables of migrate_stage: offsets, streams and (export) each record's answer type
std::vector<unsigned char> migrate_tables(const uint64_t* offsets, const uint32_t* streams, const uint32_t* types,
                                          uint32_t n) {
  std::vector<unsigned char> t((size_t)16 * n, 0);
  std::memcpy(t.data(), offsets, (size_t)8 * n);
  std::memcpy(t.data() + (size_t)8 * n, streams, (size_t)4 * n);
  if (types) std::memcpy(t.data() + (size_t)12 * n, types, (size_t)4 * n);
  return t;
}

// Record i of an import into session cs (bytes [off, off + its size) of `records`, total bytes in all): whether
// every field the unpack kernel and the next push read as a length, an index or a state is in range for cs, and the
// record's answer type and open length.  Records come from outside the program: nothing is trusted.
bool record_ok(rpl_capsule_stream* cs, const uint8_t* records, uint64_t off, uint64_t total, uint32_t* type,
               uint32_t* L) {
  rpl_ctx* c = cs->c;
  if ((off & 15u) != 0 || off > total || total - off < rpl::kRecHeaderBytes) {
    c->err = "a record offset is not a multiple of 16, or its header lies outside [0, total_bytes)";
    return false;
  }
  uint32_t h[8];
  std::memcpy(h, records + off, sizeof h);
  if (h[rpl::kRecWordMagic] != rpl::kRecMagic || h[rpl::kRecWordVersion] != rpl::kRecVersion) {
    c->err = "not a stream record of this version (magic or version)";
    return false;
  }
  if (h[rpl::kRecWordKind] != (cs->bytes ? 1u : 0u)) {
    c->err = "a record of a framed session into a byte session, or the reverse";
    return false;
  }
  const uint32_t t = h[rpl::kRecWordType];
  if (cs->types.empty() ? t != cs->ans_type : (t < RPL_ANS_MEASUREMENT || t > 0x86u)) {
    c->err = "the record's answer type is not one the destination stream decodes";
    return false;
  }
  if (h[rpl::kRecWordMaxNodes] != cs->max_nodes) {
    c->err = "the record's max_nodes differs from the session's";
    return false;
  }
  if (h[rpl::kRecWordOpen] > cs->max_nodes || (h[rpl::kRecWordFlags] & ~(rpl::kRecOpenKnown | rpl::kRecRxKnown)) != 0 ||
      h[rpl::kRecWordReserved] != 0) {
    c->err = "the record's open revolution is longer than max_nodes, or its flags are unknown";
    return false;
  }
  if (record_bytes(cs->bytes, t, h[rpl::kRecWordOpen]) > total - off) {
    c->err = "a record lies partly outside [0, total_bytes)";
    return false;
  }
  const uint8_t* held = records + off + rpl::kRecHeaderBytes;
  if (t == RPL_ANS_MEASUREMENT) {  // the byte machine's state: bytes of the unfinished record
    uint32_t state;
    std::memcpy(&state, held + 4 * rpl::kHeldOk, 4);
    if (state > 4) {
      c->err = "the record's 0x81 byte-machine state is not in 0..4";
      return false;
    }
  } else if (cs->bytes) {  // the framer's search position: bytes of the unfinished frame
    uint32_t f[2];
    std::memcpy(f, held + rpl::kRecHeldBytes + 4 * rpl::kFramerPos, sizeof f);
    static_assert(rpl::kFramerLost == rpl::kFramerPos + 1, "framer words");
    if (f[0] >= rpl_capsule_bytes(t) || f[1] > 1) {
      c->err = "the record's framer position is not below the frame size, or its lost flag is not 0 or 1";
      return false;
    }
  }
  *type = t;
  *L = h[rpl::kRecWordOpen];
  return true;
}

}  // namespace

extern "C" {

rpl_result rpl_capsule_stream_export(rpl_capsule_stream* cs, const uint32_t* streams, uint32_t n, uint8_t* records,
                                     uint64_t capacity, uint64_t* record_offsets, uint64_t* total_bytes) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if ((n && (!streams || !record_offsets)) || !total_bytes || (capacity && !records)) {
    c->err = "null streams, records, record_offsets or total_bytes";
    return RPL_RESULT_INVALID_DATA;
  }
  for (uint32_t i = 0; i < n; ++i)
    if (streams[i] >= cs->n_streams) {
      c->err = "a listed stream is not below n_streams";
      return RPL_RESULT_INVALID_DATA;
    }
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // host pushes return synchronised
  // the offsets need every listed stream's open length: read back as rpl_capsule_stream_state reads it
  std::vector<uint32_t> open(cs->n_streams), types(n);
  if (n)
    RPL_CUDA(c, cudaMemcpy(open.data(), cs->carry_len[cs->parity], (size_t)cs->n_streams * 4, cudaMemcpyDeviceToHost),
             RPL_RESULT_OPERATION_FAIL);
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; ++i) {
    types[i] = stream_type(cs, streams[i]);
    record_offsets[i] = total;
    total += record_bytes(cs->bytes, types[i], open[streams[i]]);
  }
  *total_bytes = total;
  if (total > capacity) {
    c->err = "capacity is smaller than total_bytes";
    return RPL_RESULT_INSUFFICIENT_MEMORY;
  }
  if (n == 0) return RPL_RESULT_OK;
  rpl::MigrateArgs a{};
  if (const rpl_result r = migrate_stage(cs, total, n, migrate_tables(record_offsets, streams, types.data(), n), &a);
      r != RPL_RESULT_OK)
    return r;
  a.stamps_known = cs->carry_stamped ? 1u : 0u;
  cudaStream_t st = c->lane[0].stream;
  RPL_CUDA(c, rpl::launch_stream_pack(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  RPL_CUDA(c, cudaMemcpyAsync(records, a.records, total, cudaMemcpyDeviceToHost, st), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_capsule_stream_import(rpl_capsule_stream* cs, const uint32_t* streams, uint32_t n, const uint8_t* records,
                                     const uint64_t* record_offsets, uint64_t total_bytes) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (n && (!streams || !records || !record_offsets)) {
    c->err = "null streams, records or record_offsets";
    return RPL_RESULT_INVALID_DATA;
  }
  // every record is checked before anything is written: a failure leaves the session as it was
  std::vector<uint8_t> seen(cs->n_streams, 0);
  std::vector<uint32_t> types = cs->types;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t s = streams[i];
    if (s >= cs->n_streams || seen[s]) {
      c->err = "a destination stream is not below n_streams, or is listed twice";
      return RPL_RESULT_INVALID_DATA;
    }
    seen[s] = 1;
    uint32_t t = 0, L = 0;
    if (!record_ok(cs, records, record_offsets[i], total_bytes, &t, &L)) return RPL_RESULT_INVALID_DATA;
    if (!types.empty()) types[s] = t;
  }
  if (n == 0) return RPL_RESULT_OK;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);
  rpl::MigrateArgs a{};
  if (const rpl_result r = migrate_stage(cs, total_bytes, n, migrate_tables(record_offsets, streams, nullptr, n), &a);
      r != RPL_RESULT_OK)
    return r;
  cudaStream_t st = c->lane[0].stream;
  RPL_CUDA(c, cudaMemcpyAsync(a.records, records, total_bytes, cudaMemcpyHostToDevice, st), RPL_RESULT_OPERATION_FAIL);
  if (!cs->carry_stamped) {
    // the last push kept no stamps, which made every stream's count as unknown: say so per stream, so that the
    // imported streams' stamps count at the next stamped push and the others' still do not
    RPL_CUDA(c, cudaMemsetAsync(cs->open_ts[cs->parity], 0, (size_t)cs->n_streams * 8, st), RPL_RESULT_OPERATION_FAIL);
    static_assert(rpl::kRxUnknown == ~0ull, "held_rx's unknown is all ones");
    RPL_CUDA(c, cudaMemsetAsync(cs->held_rx, 0xFF, (size_t)cs->n_streams * 8, st), RPL_RESULT_OPERATION_FAIL);
    cs->carry_stamped = true;
  }
  // The unpack writes the next push's arena (parity) alone.  The last push's views, which its clouds, nodes and
  // messages read, point into the arena it decoded into (cloud_arena, the other one), so they stay as they are.
  RPL_CUDA(c, rpl::launch_stream_unpack(a, c->num_sms, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  // records do not carry the windows over the re-gridded scans: the destinations' start over
  if (cs->win_state)
    if (const rpl_result r = windows_empty(cs, seen.data(), st); r != RPL_RESULT_OK) return r;
  if (const rpl_result r = merges_empty(cs, seen.data(), st); r != RPL_RESULT_OK) return r;  // nor the held grids
  RPL_CUDA(c, cudaStreamSynchronize(st), RPL_RESULT_OPERATION_FAIL);  // in place before any later push runs
  if (types != cs->types) return set_types(cs, std::move(types));     // a mixed session's streams take the record's type
  return RPL_RESULT_OK;
}

// ---- byte sessions: the session fed the raw serial stream (0x81: the standard-node session) ----
rpl_result rpl_capsule_stream_create_bytes(rpl_ctx* c, uint32_t ans_type, uint32_t n_streams, uint32_t stride_bytes,
                                           uint32_t max_nodes, uint32_t max_scans, rpl_capsule_stream** out) {
  if (!c || !out) return RPL_RESULT_INVALID_DATA;
  *out = nullptr;
  if (ans_type != RPL_ANS_MEASUREMENT && rpl_capsule_bytes(ans_type) == 0) {
    c->err = "a byte session takes the measurement answer types 0x81..0x86";
    return RPL_RESULT_INVALID_DATA;
  }
  return stream_create(c, ans_type, true, n_streams, stride_bytes, max_nodes, max_scans, out);
}

// ---- mixed byte sessions: an answer type per stream, switched between pushes ----
namespace {
bool answer_types_ok(rpl_ctx* c, const uint32_t* ans_types, uint32_t n_streams, const uint8_t* stream_mask) {
  if (!ans_types) {
    c->err = "null ans_types";
    return false;
  }
  for (uint32_t s = 0; s < n_streams; ++s)
    if ((!stream_mask || stream_mask[s]) && (ans_types[s] < RPL_ANS_MEASUREMENT || ans_types[s] > 0x86u)) {
      c->err = "a byte session takes the measurement answer types 0x81..0x86";
      return false;
    }
  return true;
}
}  // namespace

rpl_result rpl_capsule_stream_create_bytes_mixed(rpl_ctx* c, const uint32_t* ans_types, uint32_t n_streams,
                                                 uint32_t stride_bytes, uint32_t max_nodes, uint32_t max_scans,
                                                 rpl_capsule_stream** out) {
  if (!c || !out) return RPL_RESULT_INVALID_DATA;
  *out = nullptr;
  if (!answer_types_ok(c, ans_types, n_streams, nullptr)) return RPL_RESULT_INVALID_DATA;
  return stream_create(c, 0, true, n_streams, stride_bytes, max_nodes, max_scans, out, ans_types);
}

rpl_result rpl_capsule_stream_set_answer_types(rpl_capsule_stream* cs, const uint32_t* ans_types,
                                               const uint8_t* stream_mask) {
  if (!cs) return RPL_RESULT_INVALID_DATA;
  rpl_ctx* c = cs->c;
  if (cs->types.empty()) {
    c->err = "rpl_capsule_stream_set_answer_types needs a session made by rpl_capsule_stream_create_bytes_mixed";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!answer_types_ok(c, ans_types, cs->n_streams, stream_mask)) return RPL_RESULT_INVALID_DATA;
  // the streams whose type changes start over as the SDK's startScan leaves them: holder reset, unpacker enabled
  std::vector<uint8_t> changed(cs->n_streams, 0);
  std::vector<uint32_t> t = cs->types;
  bool any = false;
  for (uint32_t s = 0; s < cs->n_streams; ++s)
    if ((!stream_mask || stream_mask[s]) && ans_types[s] != t[s]) {
      changed[s] = 1;
      t[s] = ans_types[s];
      any = true;
    }
  if (!any) return RPL_RESULT_OK;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaEventSynchronize(cs->done), RPL_RESULT_OPERATION_FAIL);  // a push may still read the lists
  if (const rpl_result r = rpl_capsule_stream_reset(cs, changed.data()); r != RPL_RESULT_OK) return r;
  return set_types(cs, std::move(t));
}

rpl_result rpl_capsule_stream_push_bytes(rpl_capsule_stream* cs, const uint8_t* bytes, const uint32_t* byte_counts,
                                         uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                         float* intensities, uint32_t* beam_counts, float* angle_increment,
                                         uint32_t* scans_per_stream) {
  return stream_push(cs, bytes, byte_counts, sample_duration_us, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, nullptr, true, false, nullptr);
}

rpl_result rpl_capsule_stream_push_bytes_dev(rpl_capsule_stream* cs, const uint8_t* bytes, const uint32_t* byte_counts,
                                             uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                             float* intensities, uint32_t* beam_counts, float* angle_increment,
                                             uint32_t* scans_per_stream, void* stream) {
  return stream_push(cs, bytes, byte_counts, sample_duration_us, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, nullptr, true, true, stream);
}

rpl_result rpl_capsule_stream_push_bytes_ts(rpl_capsule_stream* cs, const uint8_t* bytes, const uint32_t* byte_counts,
                                            const rpl_timing* timing, uint32_t chunk_bytes, const uint64_t* chunk_rx_us,
                                            const rpl_scan_params* params, float* ranges, float* intensities,
                                            uint32_t* beam_counts, float* angle_increment, uint32_t* scans_per_stream,
                                            uint64_t* scan_begin_ts_us) {
  StampPush sp{};
  if (!stamp_args_ok(cs, params, timing, chunk_rx_us, chunk_bytes, scan_begin_ts_us, &sp)) return RPL_RESULT_INVALID_DATA;
  return stream_push(cs, bytes, byte_counts, timing ? timing->sample_duration_us : 0u, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, &sp, true, false, nullptr);
}

rpl_result rpl_capsule_stream_push_bytes_ts_dev(rpl_capsule_stream* cs, const uint8_t* bytes,
                                                const uint32_t* byte_counts, const rpl_timing* timing,
                                                uint32_t chunk_bytes, const uint64_t* chunk_rx_us,
                                                const rpl_scan_params* params, float* ranges, float* intensities,
                                                uint32_t* beam_counts, float* angle_increment,
                                                uint32_t* scans_per_stream, uint64_t* scan_begin_ts_us, void* stream) {
  StampPush sp{};
  if (!stamp_args_ok(cs, params, timing, chunk_rx_us, chunk_bytes, scan_begin_ts_us, &sp)) return RPL_RESULT_INVALID_DATA;
  return stream_push(cs, bytes, byte_counts, timing ? timing->sample_duration_us : 0u, params, ranges, intensities, beam_counts,
                     angle_increment, scans_per_stream, &sp, true, true, stream);
}

// ---- session clouds: the PointCloud2 chain over the scans the last push published, read in place ----
rpl_result rpl_capsule_stream_nodes_dev(rpl_capsule_stream* cs, uint32_t apply_ascend, const uint8_t* ascend_per_stream,
                                        rpl_node_hq* nodes, uint64_t capacity_nodes, uint64_t* node_offsets,
                                        uint32_t* node_counts, uint32_t* status, uint64_t* total_nodes, void* stream) {
  return stream_nodes_dev(cs, apply_ascend, ascend_per_stream, nodes, capacity_nodes, node_offsets, node_counts, status,
                          total_nodes, stream);
}
rpl_result rpl_capsule_stream_nodes(rpl_capsule_stream* cs, uint32_t apply_ascend, const uint8_t* ascend_per_stream,
                                    rpl_node_hq* nodes, uint64_t capacity_nodes, uint64_t* node_offsets,
                                    uint32_t* node_counts, uint32_t* status, uint64_t* total_nodes) {
  return stream_nodes(cs, apply_ascend, ascend_per_stream, nodes, capacity_nodes, node_offsets, node_counts, status,
                      total_nodes);
}
rpl_result rpl_capsule_stream_cloud_dev(rpl_capsule_stream* cs, const rpl_cloud_params* params, float* xyzi,
                                        uint32_t* point_counts, void* stream) {
  return stream_cloud_dev(cs, params, xyzi, point_counts, stream);
}

rpl_result rpl_capsule_stream_cloud(rpl_capsule_stream* cs, const rpl_cloud_params* params, float* xyzi,
                                    uint32_t* point_counts) {
  return stream_cloud(cs, params, xyzi, point_counts);
}

// ---- per-stream settings and packed messages of the last push ----------------------------------------------------
rpl_result rpl_capsule_stream_set_frames(rpl_capsule_stream* s, const char* const* frame_ids, const float* range_max) {
  return stream_set_frames(s, frame_ids, range_max);
}

rpl_result rpl_capsule_stream_set_lidars(rpl_capsule_stream* s, const rpl_lidar_settings* settings,
                                         const uint8_t* stream_mask) {
  return stream_set_lidars(s, settings, stream_mask);
}

rpl_result rpl_capsule_stream_set_clouds(rpl_capsule_stream* s, const rpl_cloud_settings* settings,
                                         const uint8_t* stream_mask) {
  return stream_set_clouds(s, settings, stream_mask);
}

rpl_result rpl_capsule_stream_set_scan_filters(rpl_capsule_stream* s, const rpl_scan_filter_settings* settings,
                                               const uint8_t* stream_mask) {
  return stream_set_scan_filters(s, settings, stream_mask);
}

rpl_result rpl_capsule_stream_set_scan_cloud_transforms(rpl_capsule_stream* s,
                                                        const rpl_scan_cloud_transform* transforms,
                                                        const char* const* target_frames, const uint8_t* stream_mask) {
  return stream_set_scan_cloud_transforms(s, transforms, target_frames, stream_mask);
}

rpl_result rpl_capsule_stream_set_scan_footprints(rpl_capsule_stream* s, const rpl_scan_footprint* footprints,
                                                  const uint8_t* stream_mask) {
  return stream_set_scan_footprints(s, footprints, stream_mask);
}

rpl_result rpl_capsule_stream_laserscan_msgs_dev(rpl_capsule_stream* s, const rpl_scan_params* params,
                                                 int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                                 uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes,
                                                 void* stream) {
  return stream_msgs_dev(s, rpl::MsgKind::kLaserScan, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                         total_bytes, stream);
}

rpl_result rpl_capsule_stream_laserscan_msgs(rpl_capsule_stream* s, const rpl_scan_params* params,
                                             int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                             uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes) {
  return stream_msgs(s, rpl::MsgKind::kLaserScan, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                     total_bytes);
}

rpl_result rpl_capsule_stream_push_laserscan_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                                  const rpl_scan_params* params, int64_t clock_offset_ns, uint8_t* msgs,
                                                  uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                                  uint64_t* total_bytes, uint32_t* scans_per_stream) {
  return push_msgs(s, in, rpl::MsgKind::kLaserScan, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                   total_bytes, scans_per_stream, false, nullptr);
}

rpl_result rpl_capsule_stream_push_laserscan_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                      const rpl_scan_params* params, int64_t clock_offset_ns,
                                                      uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                                      uint32_t* msg_sizes, uint64_t* total_bytes,
                                                      uint32_t* scans_per_stream, void* stream) {
  return push_msgs(s, in, rpl::MsgKind::kLaserScan, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                   total_bytes, scans_per_stream, true, stream);
}

rpl_result rpl_capsule_stream_push_cloud_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                              const rpl_cloud_params* params, int64_t clock_offset_ns, uint8_t* msgs,
                                              uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                              uint64_t* total_bytes, uint32_t* scans_per_stream) {
  return push_msgs(s, in, rpl::MsgKind::kPointCloud2, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                   total_bytes, scans_per_stream, false, nullptr);
}

rpl_result rpl_capsule_stream_push_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                  const rpl_cloud_params* params, int64_t clock_offset_ns,
                                                  uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                                  uint32_t* msg_sizes, uint64_t* total_bytes,
                                                  uint32_t* scans_per_stream, void* stream) {
  return push_msgs(s, in, rpl::MsgKind::kPointCloud2, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                   total_bytes, scans_per_stream, true, stream);
}

rpl_result rpl_capsule_stream_push_scan_cloud_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                                   const rpl_scan_params* scan_params,
                                                   const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                                   const rpl_msgs_out* scans, const rpl_msgs_out* clouds,
                                                   uint32_t* scans_per_stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, clouds, scans_per_stream, false,
                              nullptr);
}

rpl_result rpl_capsule_stream_push_scan_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                       const rpl_scan_params* scan_params,
                                                       const rpl_scan_cloud_params* cloud_params,
                                                       int64_t clock_offset_ns, const rpl_msgs_out* scans,
                                                       const rpl_msgs_out* clouds, uint32_t* scans_per_stream,
                                                       void* stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, clouds, scans_per_stream, true,
                              stream);
}

rpl_result rpl_capsule_stream_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_cloud_params* params,
                                             int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                             uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes,
                                             void* stream) {
  return stream_msgs_dev(s, rpl::MsgKind::kPointCloud2, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                         total_bytes, stream);
}

rpl_result rpl_capsule_stream_cloud_msgs(rpl_capsule_stream* s, const rpl_cloud_params* params, int64_t clock_offset_ns,
                                         uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                         uint64_t* total_bytes) {
  return stream_msgs(s, rpl::MsgKind::kPointCloud2, params, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                     total_bytes);
}

rpl_result rpl_capsule_stream_scan_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_scan_params* scan_params,
                                                  const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                                  uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                                  uint32_t* msg_sizes, uint64_t* total_bytes, void* stream) {
  const ScanCloudCall q{scan_params, cloud_params};
  return stream_msgs_dev(s, rpl::MsgKind::kScanCloud, &q, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                         total_bytes, stream);
}

rpl_result rpl_capsule_stream_scan_cloud_msgs(rpl_capsule_stream* s, const rpl_scan_params* scan_params,
                                              const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                              uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                              uint32_t* msg_sizes, uint64_t* total_bytes) {
  const ScanCloudCall q{scan_params, cloud_params};
  return stream_msgs(s, rpl::MsgKind::kScanCloud, &q, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                     total_bytes);
}

rpl_result rpl_capsule_stream_set_rescan_windows(rpl_capsule_stream* s, const rpl_rescan_window* windows,
                                                 const uint8_t* stream_mask) {
  return stream_set_rescan_windows(s, windows, stream_mask);
}

rpl_result rpl_capsule_stream_push_rescan_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                               const rpl_scan_params* scan_params,
                                               const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                               const rpl_msgs_out* scans, const rpl_msgs_out* rescans,
                                               uint32_t* scans_per_stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, rescans, scans_per_stream, false,
                              nullptr, true);
}

rpl_result rpl_capsule_stream_push_rescan_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                   const rpl_scan_params* scan_params,
                                                   const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                                   const rpl_msgs_out* scans, const rpl_msgs_out* rescans,
                                                   uint32_t* scans_per_stream, void* stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, rescans, scans_per_stream, true,
                              stream, true);
}

rpl_result rpl_capsule_stream_set_rescan_merges(rpl_capsule_stream* s, const uint32_t* group_of_stream,
                                                const uint32_t* max_age, uint32_t n_groups) {
  return stream_set_rescan_merges(s, group_of_stream, max_age, n_groups);
}

rpl_result rpl_capsule_stream_push_rescan_merge_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                                     const rpl_scan_params* scan_params,
                                                     const rpl_scan_cloud_params* cloud_params,
                                                     int64_t clock_offset_ns, const rpl_msgs_out* scans,
                                                     const rpl_msgs_out* rescans, const rpl_msgs_out* merged,
                                                     uint32_t* scans_per_stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, rescans, scans_per_stream, false,
                              nullptr, true, true, merged);
}

rpl_result rpl_capsule_stream_push_rescan_merge_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                         const rpl_scan_params* scan_params,
                                                         const rpl_scan_cloud_params* cloud_params,
                                                         int64_t clock_offset_ns, const rpl_msgs_out* scans,
                                                         const rpl_msgs_out* rescans, const rpl_msgs_out* merged,
                                                         uint32_t* scans_per_stream, void* stream) {
  return push_scan_cloud_msgs(s, in, scan_params, cloud_params, clock_offset_ns, scans, rescans, scans_per_stream, true,
                              stream, true, true, merged);
}

rpl_result rpl_capsule_stream_set_rescans(rpl_capsule_stream* s, const rpl_rescan_settings* settings,
                                          const uint8_t* stream_mask) {
  return stream_set_rescans(s, settings, stream_mask);
}

rpl_result rpl_capsule_stream_rescan_msgs_dev(rpl_capsule_stream* s, const rpl_scan_params* scan_params,
                                              const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                              uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                              uint32_t* msg_sizes, uint64_t* total_bytes, void* stream) {
  const ScanCloudCall q{scan_params, cloud_params};
  return stream_msgs_dev(s, rpl::MsgKind::kRescan, &q, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                         total_bytes, stream);
}

rpl_result rpl_capsule_stream_rescan_msgs(rpl_capsule_stream* s, const rpl_scan_params* scan_params,
                                          const rpl_scan_cloud_params* cloud_params, int64_t clock_offset_ns,
                                          uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                          uint64_t* total_bytes) {
  const ScanCloudCall q{scan_params, cloud_params};
  return stream_msgs(s, rpl::MsgKind::kRescan, &q, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                     total_bytes);
}

// ---- LaserScan / PointCloud2 -> CDR (SURVEY.md 8(f) rank 3) -------------------------------------
namespace {
struct CdrWriter {  // XCDR1 little endian; alignment counts from the byte after the encapsulation header
  uint8_t* b;
  uint32_t n = 0;
  explicit CdrWriter(uint8_t* buf) : b(buf) {
    const uint8_t enc[4] = {0x00, 0x01, 0x00, 0x00};
    std::memcpy(b, enc, 4);
    n = 4;
  }
  void align(uint32_t a) {
    while ((n - 4) % a) b[n++] = 0;
  }
  void u32(uint32_t v) {
    align(4);
    std::memcpy(b + n, &v, 4);
    n += 4;
  }
  void u8(uint8_t v) { b[n++] = v; }
  void str(const char* s, uint32_t len) {
    u32(len + 1);
    std::memcpy(b + n, s, len);
    n += len;
    b[n++] = 0;
  }
};
uint32_t header_bytes(uint32_t frame_id_len) { return 4 + ((12 + frame_id_len + 1 + 3) & ~3u); }
}  // namespace

uint32_t rpl_laserscan_cdr_size(uint32_t frame_id_len, uint32_t beam_count) {
  return header_bytes(frame_id_len) + 28 + 4 + 4 * beam_count + 4 + 4 * beam_count;
}

uint32_t rpl_pointcloud2_cdr_size(uint32_t frame_id_len, uint32_t n_points) {
  // height, width, fields count; x/y/z (20 bytes each), intensity (28); is_bigendian + pad; point_step,
  // row_step, data length; data; is_dense
  return header_bytes(frame_id_len) + 12 + 3 * 20 + 28 + 4 + 12 + 16 * n_points + 1;
}

rpl_result rpl_laserscan_cdr_batch_dev(rpl_ctx* c, const rpl_laserscan_meta* meta, const float* angle_increment,
                                       const char* frame_id, const float* ranges, const float* intensities,
                                       const uint32_t* beam_counts, uint32_t n_scans, uint32_t stride,
                                       uint8_t* cdr_out, uint32_t cdr_stride, uint32_t* cdr_sizes, void* stream) {
  if (!c || !meta || !frame_id || !ranges || !intensities || !beam_counts || !cdr_out) return RPL_RESULT_INVALID_DATA;
  const size_t L = std::strlen(frame_id);
  if (!frame_id_length_ok(c, L)) return RPL_RESULT_INVALID_DATA;
  if ((cdr_stride & 3u) || cdr_stride < rpl_laserscan_cdr_size((uint32_t)L, stride) ||
      (reinterpret_cast<uintptr_t>(cdr_out) & 3u)) {
    c->err = "cdr_out must be 4-byte aligned, cdr_stride a multiple of 4 and >= rpl_laserscan_cdr_size(len, stride)";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_scans == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::CdrTemplate t{};
  CdrWriter w(t.prefix);
  w.u32(0);  // stamp.sec     (patched)
  w.u32(0);  // stamp.nanosec (patched)
  w.str(frame_id, (uint32_t)L);
  for (int i = 0; i < 7; ++i) w.u32(0);  // angle_min .. range_max (patched)
  w.u32(0);                              // ranges count (patched)
  t.prefix_bytes = w.n;
  rpl::LaserScanCdrArgs a{};
  a.meta = reinterpret_cast<const rpl::LaserScanMeta*>(meta);
  a.angle_increment = angle_increment;
  a.ranges = ranges;
  a.intensities = intensities;
  a.beam_counts = beam_counts;
  a.n_scans = n_scans;
  a.stride = stride;
  a.cdr_out = cdr_out;
  a.cdr_stride = cdr_stride;
  a.cdr_sizes = cdr_sizes;
  RPL_CUDA(c, rpl::launch_laserscan_cdr(a, t, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

rpl_result rpl_pointcloud2_cdr_batch_dev(rpl_ctx* c, const uint32_t* stamps, const char* frame_id,
                                         const float* xyzi, const uint32_t* point_counts, uint32_t n_clouds,
                                         uint32_t stride, uint8_t* cdr_out, uint32_t cdr_stride,
                                         uint32_t* cdr_sizes, void* stream) {
  if (!c || !stamps || !frame_id || !xyzi || !point_counts || !cdr_out) return RPL_RESULT_INVALID_DATA;
  const size_t L = std::strlen(frame_id);
  if (!frame_id_length_ok(c, L)) return RPL_RESULT_INVALID_DATA;
  if ((cdr_stride & 15u) || cdr_stride < rpl_pointcloud2_cdr_size((uint32_t)L, stride) ||
      (reinterpret_cast<uintptr_t>(cdr_out) & 15u)) {
    c->err = "cdr_out must be 16-byte aligned, cdr_stride a multiple of 16 and >= rpl_pointcloud2_cdr_size(len, stride)";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_clouds == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::CdrTemplate t{};
  CdrWriter w(t.prefix);
  w.u32(0);
  w.u32(0);
  w.str(frame_id, (uint32_t)L);
  w.u32(1);  // height
  w.align(4);
  t.patch_width = w.n;
  w.u32(0);  // width (patched)
  w.u32(4);  // fields
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (uint32_t f = 0; f < 4; ++f) {
    w.str(names[f], (uint32_t)std::strlen(names[f]));
    w.u32(4 * f);  // offset
    w.u8(7);       // datatype FLOAT32
    w.u32(1);      // count
  }
  w.u8(0);         // is_bigendian
  w.u32(16);       // point_step
  w.align(4);
  t.patch_row_step = w.n;
  w.u32(0);        // row_step (patched)
  w.u32(0);        // data length (patched)
  t.prefix_bytes = w.n;
  rpl::PointCloudCdrArgs a{};
  a.stamps = stamps;
  a.xyzi = xyzi;
  a.point_counts = point_counts;
  a.n_clouds = n_clouds;
  a.stride = stride;
  a.cdr_out = cdr_out;
  a.cdr_stride = cdr_stride;
  a.cdr_sizes = cdr_sizes;
  RPL_CUDA(c, rpl::launch_pointcloud2_cdr(a, t, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// ---- per-sample timestamps (SURVEY.md 8(f) rank 4) ----------------------------------------------
rpl_result rpl_node_timestamps_dev(rpl_ctx* c, uint32_t ans_type, const rpl_timing* timing,
                                   const uint64_t* capsule_rx_us, const uint32_t* capsule_status,
                                   const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                   uint32_t n_streams, uint32_t stride_capsules, uint64_t* node_ts_us, void* stream) {
  if (!c || !timing || !capsule_rx_us || !capsule_status || !capsule_node_offset || !capsule_counts || !node_ts_us)
    return RPL_RESULT_INVALID_DATA;
  if (misaligned8(capsule_rx_us) || misaligned8(node_ts_us)) {
    c->err = "timestamp buffers must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (capsule_bytes(c, ans_type) == 0) return RPL_RESULT_INVALID_DATA;
  if (n_streams == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::TimingDesc t{timing->sample_duration_us, timing->native_baudrate, timing->linkage_delay_us,
                    timing->native_interface_type};
  rpl::TimestampArgs a{};
  a.capsule_rx_us = reinterpret_cast<const unsigned long long*>(capsule_rx_us);
  a.capsule_status = capsule_status;
  a.capsule_node_offset = capsule_node_offset;
  a.capsule_counts = capsule_counts;
  a.n_streams = n_streams;
  a.stride_capsules = stride_capsules;
  a.node_ts_us = reinterpret_cast<unsigned long long*>(node_ts_us);
  RPL_CUDA(c, rpl::launch_node_timestamps(ans_type, t, a, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

rpl_result rpl_normal_timestamps_dev(rpl_ctx* c, const rpl_timing* timing, const uint32_t* node_end,
                                     const uint32_t* node_counts, uint32_t n_streams, uint32_t stride_nodes,
                                     uint32_t chunk_bytes, const uint64_t* chunk_rx_us, uint32_t stride_chunks,
                                     uint64_t* node_ts_us, void* stream) {
  if (!c || !timing || !node_end || !node_counts || !chunk_rx_us || !node_ts_us || chunk_bytes == 0)
    return RPL_RESULT_INVALID_DATA;
  if (misaligned8(chunk_rx_us) || misaligned8(node_ts_us)) {
    c->err = "timestamp buffers must be 8-byte aligned";
    return RPL_RESULT_INVALID_DATA;
  }
  if (n_streams == 0) return RPL_RESULT_OK;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::TimingDesc t{timing->sample_duration_us, timing->native_baudrate, timing->linkage_delay_us,
                    timing->native_interface_type};
  rpl::NormalTimestampArgs a{};
  a.node_end = node_end;
  a.node_counts = node_counts;
  a.n_streams = n_streams;
  a.stride_nodes = stride_nodes;
  a.chunk_bytes = chunk_bytes;
  a.stride_chunks = stride_chunks;
  a.chunk_rx_us = reinterpret_cast<const unsigned long long*>(chunk_rx_us);
  a.node_ts_us = reinterpret_cast<unsigned long long*>(node_ts_us);
  RPL_CUDA(c, rpl::launch_normal_timestamps(t, a, st), RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// ---- synthetic streams ------------------------------------------------------------------------
rpl_result rpl_synth_batch_dev(rpl_ctx* c, uint64_t first_scan_id, uint32_t n_scans, uint32_t n,
                               uint32_t stride, int variant, rpl_node_hq* nodes, uint32_t* counts,
                               void* stream) {
  if (!c || !nodes || n > stride || variant < 0 || variant > 4) return RPL_RESULT_INVALID_DATA;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  RPL_CUDA(c, rpl::launch_synth(first_scan_id, n_scans, n, stride, variant,
                                reinterpret_cast<uint2*>(nodes), counts, st),
           RPL_RESULT_OPERATION_FAIL);
  c->launches++;
  return RPL_RESULT_OK;
}

// ---- PointCloud2 path ----------------------------------------------------------------------------
rpl_result rpl_cloud_batch_dev(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                               uint32_t n_scans, uint32_t stride, const rpl_cloud_params* params,
                               float* xyzi, uint32_t* point_counts, void* stream) {
  return rpl_cloud_footprint_batch_dev(c, nodes, counts, n_scans, stride, params, nullptr, xyzi, point_counts, stream);
}

rpl_result rpl_cloud_footprint_batch_dev(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                                         uint32_t n_scans, uint32_t stride, const rpl_cloud_params* params,
                                         const rpl_scan_footprint* footprint, float* xyzi, uint32_t* point_counts,
                                         void* stream) {
  if (!c || !nodes || !counts || !params || !xyzi || !point_counts) return RPL_RESULT_INVALID_DATA;
  if (footprint && !scan_footprint_ok(c, *footprint)) return RPL_RESULT_INVALID_DATA;
  if (n_scans == 0) return RPL_RESULT_OK;
  if (n_scans > c->max_scans) {
    c->err = "n_scans exceeds max_scans";
    return RPL_RESULT_INVALID_DATA;
  }
  if (!cloud_params_ok(c, params)) return RPL_RESULT_INVALID_DATA;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  rpl::ScanBatchArgs a{};
  a.nodes = reinterpret_cast<const uint2*>(nodes);
  a.counts = counts;
  a.n_scans = n_scans;
  a.stride = stride;
  a.beam_counts = point_counts;  // points kept per scan
  a.fallback_list = c->lane[0].fallback_list;
  a.is_new_protocol = params->is_new_protocol;
  a.xyzi = reinterpret_cast<float4*>(xyzi);
  a.trig = c->lane[0].cws.trig;
  a.angle = c->lane[0].cws.angle;
  a.range_min = params->range_min;
  a.range_max = params->range_max;
  a.intensity_min = params->intensity_min;
  // Revolutions of at most 4096 nodes: the whole chain (window, xyz, SOR, voxel grid) in one kernel, in shared
  // memory (scan_small.cu); the separate in-place post passes then only see the duplicate-key scans that kernel
  // handed to the general kernel.  Larger revolutions: steps 1-3 inside the scan kernels, steps 4-5 as post passes.
  // A footprint with polygons: steps 1-3 in the scan kernels, the footprint pass, then steps 4-5 over every scan.
  rpl::ScanFootprint one{};
  if (footprint) one = scan_footprint_entry(*footprint);
  const bool fp = one.n_polygons != 0;
  bool fused = false;
  const uint32_t flags = (params->flags & RPL_CLOUD_NO_FUSED) ? RPL_FLAG_NO_SMALL : 0u;
  rpl_result r = scratch_enter(c, c->lane[0], st);
  if (r == RPL_RESULT_OK) r = enqueue_args(c, c->lane[0], a, flags, st, fp ? nullptr : params, &fused);
  if (r == RPL_RESULT_OK && fp) r = footprint_clouds(c, a, nullptr, one, point_counts, st);
  if (r != RPL_RESULT_OK) return r;
  if (params->sor_k > 0 || params->voxel_size > 0.0f) {
    int launched = 0;
    RPL_CUDA(c, rpl::launch_cloud_post(a.xyzi, point_counts, n_scans, stride, params->sor_k, params->sor_alpha,
                                       params->voxel_size, c->lane[0].cws, fused ? a.fallback_list : nullptr,
                                       fused ? c->lane[0].hand_off_count() : nullptr, st, &launched),
             RPL_RESULT_OPERATION_FAIL);
    c->launches += launched;
  }
  return scratch_leave(c, c->lane[0], st);
}

rpl_result rpl_cloud_batch(rpl_ctx* c, const rpl_node_hq* nodes, const uint32_t* counts,
                           uint32_t n_scans, uint32_t stride, const rpl_cloud_params* params,
                           float* xyzi, uint32_t* point_counts) {
  if (!c || !nodes || !counts || !params || !xyzi || !point_counts) return RPL_RESULT_INVALID_DATA;
  if (n_scans == 0) return RPL_RESULT_OK;
  if (n_scans > c->max_scans) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  Lane& l = c->lane[0];
  const size_t cnt = (size_t)n_scans * stride;
  struct Regions { rpl_node_hq* nodes; float* xyzi; uint32_t *counts, *pcount; };
  auto layout = [&](Carve& k) {
    return Regions{k.take<rpl_node_hq>(cnt), k.take<float>(cnt * 4), k.take<uint32_t>(n_scans),
                   k.take<uint32_t>(n_scans)};
  };
  rpl_result r = grow_stage(c, 1, layout);
  if (r != RPL_RESULT_OK) return r;
  Carve k{l.stage};
  const Regions d = layout(k);
  RPL_CUDA(c, cudaMemcpyAsync(d.nodes, nodes, cnt * sizeof(rpl_node_hq), cudaMemcpyHostToDevice, l.stream),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(d.counts, counts, n_scans * sizeof(uint32_t), cudaMemcpyHostToDevice, l.stream),
           RPL_RESULT_OPERATION_FAIL);
  r = rpl_cloud_batch_dev(c, d.nodes, d.counts, n_scans, stride, params, d.xyzi, d.pcount, l.stream);
  if (r != RPL_RESULT_OK) return r;
  RPL_CUDA(c, cudaMemcpyAsync(xyzi, d.xyzi, cnt * 4 * sizeof(float), cudaMemcpyDeviceToHost, l.stream),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaMemcpyAsync(point_counts, d.pcount, n_scans * sizeof(uint32_t), cudaMemcpyDeviceToHost, l.stream),
           RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaStreamSynchronize(l.stream), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_cloud_fuse_dev(rpl_ctx* c, const float* xyzi, const uint32_t* point_counts,
                              uint32_t n_scans, uint32_t stride, float* fused, uint32_t* offsets,
                              uint32_t* total, void* stream) {
  if (!c || !xyzi || !point_counts || !fused || !offsets || !total) return RPL_RESULT_INVALID_DATA;
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  int launched = 0;
  RPL_CUDA(c, rpl::launch_cloud_fuse(reinterpret_cast<const float4*>(xyzi), point_counts, n_scans, stride,
                                     reinterpret_cast<float4*>(fused), 0xFFFFFFFFu, offsets, total, st, &launched),
           RPL_RESULT_OPERATION_FAIL);
  c->launches += launched;
  return RPL_RESULT_OK;
}

// ---- peer memory: fuse + all-gather in one kernel (SURVEY.md 8(e)) ---------------------------------
size_t rpl_peer_gather_bytes(uint32_t world, uint32_t slot_points) {
  return (size_t)rpl::kPeerHeaderBytes + (size_t)world * slot_points * 16;
}

rpl_result rpl_peer_alloc(rpl_ctx* c, size_t bytes, void** dev_ptr, uint8_t* handle_out) {
  if (!c || !dev_ptr || !handle_out || bytes == 0) return RPL_RESULT_INVALID_DATA;
  static_assert(sizeof(cudaIpcMemHandle_t) == RPL_IPC_HANDLE_BYTES, "IPC handle size");
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  void* p = nullptr;
  RPL_CUDA(c, cudaMalloc(&p, bytes), RPL_RESULT_INSUFFICIENT_MEMORY);
  cudaIpcMemHandle_t h;
  if (!cuda_ok(c, cudaMemset(p, 0, bytes), "cudaMemset") || !cuda_ok(c, cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle")) {
    cudaFree(p);
    return RPL_RESULT_OPERATION_FAIL;
  }
  std::memcpy(handle_out, &h, sizeof(h));
  *dev_ptr = p;
  return RPL_RESULT_OK;
}

rpl_result rpl_peer_open(rpl_ctx* c, const uint8_t* handle, void** peer_ptr) {
  if (!c || !handle || !peer_ptr) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, sizeof(h));
  RPL_CUDA(c, cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_peer_close(rpl_ctx* c, void* peer_ptr) {
  if (!c || !peer_ptr) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaIpcCloseMemHandle(peer_ptr), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_peer_free(rpl_ctx* c, void* dev_ptr) {
  if (!c || !dev_ptr) return RPL_RESULT_INVALID_DATA;
  RPL_CUDA(c, cudaSetDevice(c->device), RPL_RESULT_OPERATION_FAIL);
  RPL_CUDA(c, cudaFree(dev_ptr), RPL_RESULT_OPERATION_FAIL);
  return RPL_RESULT_OK;
}

rpl_result rpl_cloud_fuse_push_dev(rpl_ctx* c, const float* xyzi, const uint32_t* point_counts, uint32_t n_scans,
                                   uint32_t stride, void* const* peer_bases, uint32_t world, uint32_t rank,
                                   uint32_t slot_points, uint32_t* offsets, uint32_t* total, void* stream) {
  if (!c || !xyzi || !point_counts || !peer_bases || !offsets || !total) return RPL_RESULT_INVALID_DATA;
  if (world == 0 || world > rpl::kMaxPeers || rank >= world) {
    c->err = "world must be in [1, 16] and rank < world";
    return RPL_RESULT_INVALID_DATA;
  }
  rpl::PeerBases peers{};
  for (uint32_t p = 0; p < world; ++p) {
    if (!peer_bases[p] || (reinterpret_cast<uintptr_t>(peer_bases[p]) & 15u)) {
      c->err = "peer buffers must be non-null and 16-byte aligned";
      return RPL_RESULT_INVALID_DATA;
    }
    peers.base[p] = static_cast<unsigned char*>(peer_bases[p]);
  }
  cudaStream_t st;
  if (!enter_device(c, stream, &st)) return RPL_RESULT_OPERATION_FAIL;
  int launched = 0;
  RPL_CUDA(c, rpl::launch_cloud_fuse_push(reinterpret_cast<const float4*>(xyzi), point_counts, n_scans, stride, peers,
                                          world, rank, slot_points, offsets, total, st, &launched),
           RPL_RESULT_OPERATION_FAIL);
  c->launches += launched;
  return RPL_RESULT_OK;
}

}  // extern "C"
