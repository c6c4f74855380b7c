/* include/rpl_b200.h -- C-ABI of librplidar_b200.so (the drop-in boundary).
 *
 * H100-native (sm_90a) replacement for the per-scan point-processing hot path of
 * frozenreboot/rplidar_ros2_driver.  Every entry point is extern "C", POD-only, caller owns
 * all memory, nothing throws across the boundary, and results are sl_result-style uint32_t
 * (reference src/sdk/include/sl_types.h:70-81).  There is NO CPU fallback: without a CUDA
 * device rpl_ctx_create fails and nothing else can be called.
 *
 * What each entry point replaces in the reference:
 *
 *   rpl_ascend_scan          sl::ILidarDriver::ascendScanData(node*, count)
 *                              src/sdk/include/sl_lidar_driver.h:477
 *                              (body src/sdk/src/sl_lidar_driver.cpp:128-184, entry :957-960)
 *   rpl_laserscan            the compute body of RPlidarNode::publish_scan
 *                              src/rplidar_node.cpp:581-677 (filter+unpack :581-600, sort
 *                              :605-607, Mode A :630-660, Mode B :661-677)
 *   rpl_scan                 both, fused: RealLidarDriver::grab_scan_data's "ascend if the
 *                              profile asks" (src/lidar_driver_wrapper.cpp:328-329) followed by
 *                              publish_scan -- one host<->device round trip per scan
 *   rpl_*_batch              the same per scan over [n_scans][stride] buffers (the reference
 *                              has no batched form: one scan thread per node,
 *                              src/rplidar_node.cpp:220)
 *   rpl_*_batch_dev          the batched forms on buffers already resident in HBM
 *   rpl_cloud_batch[_dev]    north-star extensions with no reference counterpart (polar->xyz
 *                              PointCloud2 packing, range/intensity window, statistical
 *                              outlier removal, voxel grid); defined by oracle/cloud_oracle.cpp
 *   rpl_synth_batch_dev      synthetic scan streams of SURVEY.md 8(d) generated in HBM
 *
 * and, either side of that path (SURVEY.md 8(f)):
 *
 *   rpl_decode_*             the SDK's sample-data unpackers, all six measurement answer types
 *                              src/sdk/src/dataunpacker/unpacker/handler_{capsules,normalnode,hqnode}.cpp
 *   rpl_node_timestamps_dev  the timestamp the unpackers attach to every node (_getSampleDelayOffsetIn*Mode)
 *   rpl_assemble_scans_dev   ScanDataHolder::pushScanNodeData / rewindCurrentScanData
 *                              src/sdk/src/sl_lidar_driver.cpp:272-315
 *   rpl_capsule_stream_*     the capsule unpackers (express, HQ, ultra, dense, ultra-dense) and the ScanDataHolder
 *                              as live, per-stream state across calls: wire capsules pushed in any pieces publish the
 *                              scans of the whole stream; rpl_capsule_stream_*_bytes: the raw serial bytes in any
 *                              pieces, with the unpackers' search for the sync bytes carried across calls, and for
 *                              the standard-node unpacker the raw 0x81 bytes
 *   rpl_capsule_stream_push*_ts*  a session push that also stamps every published scan with its scan-begin time
 *   rpl_capsule_stream_*_msgs*    (with rpl_capsule_stream_set_frames) the serialised LaserScan / PointCloud2 of every
 *                              scan a session push published, packed: what scan_pub_->publish hands the RMW layer
 *                              src/rplidar_node.cpp:616-679
 *   rpl_*_cdr_batch_dev      the serialised form of the message scan_pub_->publish hands to the RMW layer
 *                              src/rplidar_node.cpp:679
 *   rpl_cloud_fuse_push_dev  (with rpl_peer_*) the fused cloud's all-gather across GPUs, in the pack kernel
 *
 * Buffer contract of the *_dev entry points: every count array entry must be <= its stride (counts are
 * read on the device and not clamped), device pointers must belong to the context's device, and work is
 * ordered on the stream passed in (NULL = the context's own stream).  The context's own stream is a non-blocking
 * stream: it does not wait for work the caller has in flight on other streams (the legacy default stream included).
 * A caller that fills its device buffers on a stream of its own either passes that stream, or synchronises before the
 * call and calls rpl_ctx_synchronize before it reads the results.  One context's calls may be issued on several
 * streams, device and host calls mixed: their scan kernels take turns on the context's scan scratch in the order the
 * calls were made (each call waits on its stream for the previous call's scan kernels), so every call gives what it
 * gives alone.
 *
 * Tie rule.  The reference sorts with std::sort (unstable); on equal angle_z_q14 its order
 * is whatever libstdc++'s introsort produces.  This library defines the order: equal keys
 * keep buffer order (stable).  On tie-free scans results are bit-identical to the reference.
 *
 * Threading (reference: one scan thread holding driver_mutex_, src/rplidar_node.cpp:420-439):
 * a context is single-threaded; use one context per thread.  No global state.
 */
#ifndef RPL_B200_H_
#define RPL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RPL_ABI_VERSION 1u

typedef uint32_t rpl_result;
/* reference src/sdk/include/sl_types.h:72-81 */
#define RPL_RESULT_OK 0u
#define RPL_RESULT_FAIL_BIT 0x80000000u
#define RPL_RESULT_INVALID_DATA 0x80008000u
#define RPL_RESULT_OPERATION_FAIL 0x80008001u
#define RPL_RESULT_OPERATION_TIMEOUT 0x80008002u
#define RPL_RESULT_OPERATION_NOT_SUPPORT 0x80008004u
#define RPL_RESULT_INSUFFICIENT_MEMORY 0x80008006u
#define RPL_IS_OK(x) (((x) & RPL_RESULT_FAIL_BIT) == 0u)

/* reference src/sdk/include/sl_lidar_cmd.h:272-278 (sizeof 8, offsets 0/2/6/7) */
typedef struct __attribute__((packed)) rpl_node_hq {
  uint16_t angle_z_q14; /* 90 deg / 16384 per unit; 65536 = 360 deg */
  uint32_t dist_mm_q2;  /* quarter millimetres; 0 = no measurement   */
  uint8_t quality;
  uint8_t flag;         /* bit0 = scan start sync (sl_lidar_cmd.h:178) */
} rpl_node_hq;

typedef struct rpl_scan_params {
  uint8_t is_new_protocol; /* intensity = quality (1) or quality>>2 (0); rplidar_node.cpp:575-590 */
  uint8_t scan_processing; /* 1 = Mode A resample, 0 = Mode B raw map; rplidar_node.cpp:630 */
  uint8_t inverted;        /* rplidar_node.cpp:644,673 */
  uint8_t apply_ascend;    /* angle_compensate; lidar_driver_wrapper.cpp:107,328 */
  uint32_t flags;          /* RPL_FLAG_* */
} rpl_scan_params;

#define RPL_FLAG_FORCE_GENERAL 1u /* route every scan through the general (radix-sort) kernel */
#define RPL_FLAG_NO_TMA 2u        /* use the register-streamed fast kernel (scan_fast.cu) even when the
                                     TMA-ring kernel (scan_tma.cu) applies; for A/B measurements */
#define RPL_FLAG_NO_SMALL 4u      /* do not use the shared-memory-resident kernels (scan_small.cu) for
                                     revolutions of at most 8192 nodes; for A/B measurements */
#define RPL_FLAG_PER_STREAM 8u    /* stream sessions: every stream's own rpl_lidar_settings (rpl_capsule_stream_set_lidars)
                                     instead of this struct's settings and the push's timing; other calls ignore it */

/* per-scan path report (optional output) */
#define RPL_PATH_FAST 0u    /* tie-free scan: bitmap-rank kernel */
#define RPL_PATH_GENERAL 1u /* duplicate keys (or forced): stable radix-sort kernel */

typedef struct rpl_cloud_params {
  float range_min;     /* keep range_min <= r <= range_max */
  float range_max;
  float intensity_min; /* keep intensity >= intensity_min */
  float voxel_size;    /* metres; 0 disables the voxel grid */
  uint32_t sor_k;      /* 0 disables statistical outlier removal; <= 32 */
  float sor_alpha;
  uint8_t is_new_protocol;
  uint8_t flags;       /* RPL_CLOUD_* */
  uint8_t pad[2];
} rpl_cloud_params;
#define RPL_CLOUD_NO_FUSED 1u /* run SOR / voxel grid as separate passes even where the shared-memory kernel
                                 could fuse them (A/B measurements, second implementation for the tests) */
#define RPL_CLOUD_PER_STREAM 2u /* stream sessions: every stream's own is_new_protocol (rpl_capsule_stream_set_lidars) for
                                   the intensity and the intensity_min window; other calls ignore it */
#define RPL_CLOUD_PER_STREAM_CHAIN 4u /* stream sessions: every stream's own chain (rpl_capsule_stream_set_clouds) in
                                         place of this struct's range_min .. sor_alpha; other calls ignore it */

typedef struct rpl_ctx rpl_ctx;

/* ---- context -------------------------------------------------------------------------- */
uint32_t rpl_abi_version(void);
/* device: CUDA ordinal.  max_nodes: largest scan (nodes) the context will see; max_scans:
 * largest batch for the HOST-buffer entry points (device staging is sized from these). */
rpl_result rpl_ctx_create(int device, uint32_t max_nodes, uint32_t max_scans, rpl_ctx** out);
void rpl_ctx_destroy(rpl_ctx* ctx);
const char* rpl_last_error(const rpl_ctx* ctx);
/* Block until everything queued by this context has finished. */
rpl_result rpl_ctx_synchronize(rpl_ctx* ctx);
/* Pinned host memory for the host-buffer entry points (optional; pageable works, slower). */
rpl_result rpl_host_alloc(size_t bytes, void** out);
void rpl_host_free(void* p);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
uint64_t rpl_ctx_launch_count(const rpl_ctx* ctx);
/* Kernel timing for roofline reports: when enabled, every scan-kernel launch is bracketed by
 * CUDA events on the stream it is launched on.  rpl_ctx_profile_read synchronises, returns
 * the summed durations (ms) and launch counts since the last read, and clears them. */
rpl_result rpl_ctx_profile(rpl_ctx* ctx, int enable);
rpl_result rpl_ctx_profile_read(rpl_ctx* ctx, double* fast_ms, uint32_t* fast_launches,
                                double* general_ms, uint32_t* general_launches);

/* ---- single scan, host buffers (the reference-shaped calls) --------------------------- */
/* In place, like ascendScanData.  RPL_RESULT_OPERATION_FAIL when no node is measured
 * (buffer untouched) or count == 0. */
rpl_result rpl_ascend_scan(rpl_ctx* ctx, rpl_node_hq* nodes, size_t count);
/* ranges / intensities: `count` floats each; the first *beam_count are written.
 * *beam_count == 0 means the reference would not publish (no measured node). */
rpl_result rpl_laserscan(rpl_ctx* ctx, const rpl_node_hq* nodes, size_t count,
                         const rpl_scan_params* params, float* ranges, float* intensities,
                         uint32_t* beam_count, float* angle_increment);
/* Fused grab_scan_data glue + publish_scan: nodes are ascended in place when
 * params->apply_ascend (its sl_result goes to *ascend_status, may be NULL), then converted. */
rpl_result rpl_scan(rpl_ctx* ctx, rpl_node_hq* nodes, size_t count, const rpl_scan_params* params,
                    float* ranges, float* intensities, uint32_t* beam_count,
                    float* angle_increment, rpl_result* ascend_status);

/* ---- batches, host buffers ------------------------------------------------------------ */
/* nodes: [n_scans][stride]; counts[s] <= stride nodes are live in scan s.
 * nodes_out (may be NULL, may equal nodes): ascended node buffers, same layout.
 * ranges/intensities: [n_scans][stride] floats; beam_counts/angle_increment/status/path:
 * [n_scans] (each may be NULL).  status[s] = ascendScanData's sl_result when apply_ascend,
 * else RPL_RESULT_OK. */
rpl_result rpl_scan_batch(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* counts,
                          uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                          rpl_node_hq* nodes_out, float* ranges, float* intensities,
                          uint32_t* beam_counts, float* angle_increment, uint32_t* status,
                          uint32_t* path);
rpl_result rpl_ascend_scan_batch(rpl_ctx* ctx, rpl_node_hq* nodes, const uint32_t* counts,
                                 uint32_t n_scans, uint32_t stride, uint32_t* status);
rpl_result rpl_laserscan_batch(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* counts,
                               uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                               float* ranges, float* intensities, uint32_t* beam_counts,
                               float* angle_increment);

/* ---- batches, device buffers (asynchronous on `stream`, a cudaStream_t; NULL = the
 * context's own stream).  Same layout as above; nodes_out must not alias nodes. ---------- */
rpl_result rpl_scan_batch_dev(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* counts,
                              uint32_t n_scans, uint32_t stride, const rpl_scan_params* params,
                              rpl_node_hq* nodes_out, float* ranges, float* intensities,
                              uint32_t* beam_counts, float* angle_increment, uint32_t* status,
                              uint32_t* path, void* stream);

/* ---- PointCloud2 path (extensions; oracle/cloud_oracle.cpp is the definition) --------- */
/* xyzi: [n_scans][stride][4] floats (x, y, z, intensity = PointCloud2 point_step 16);
 * point_counts[s] = points written for scan s. */
rpl_result rpl_cloud_batch_dev(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* counts,
                               uint32_t n_scans, uint32_t stride, const rpl_cloud_params* params,
                               float* xyzi, uint32_t* point_counts, void* stream);
rpl_result rpl_cloud_batch(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* counts,
                           uint32_t n_scans, uint32_t stride, const rpl_cloud_params* params,
                           float* xyzi, uint32_t* point_counts);
/* Packs the per-scan clouds of a batch into one dense cloud (the per-GPU "fused cloud" that
 * is all-gathered across ranks): fused[0..*total) points, 16 B each; offsets[s] = first point
 * of scan s.  fused must hold n_scans*stride points.  n_scans == 0 is an empty cloud: *total = 0. */
rpl_result rpl_cloud_fuse_dev(rpl_ctx* ctx, const float* xyzi, const uint32_t* point_counts,
                              uint32_t n_scans, uint32_t stride, float* fused, uint32_t* offsets,
                              uint32_t* total, void* stream);

/* ---- fuse + all-gather through peer memory (SURVEY.md 8(e): one process per GPU, NVLink P2P) ---- */
/* rpl_cloud_fuse_dev + one NCCL all-gather writes the dense cloud locally and lets the collective read
 * it again.  rpl_cloud_fuse_push_dev does both in ONE kernel: every point is stored straight into slot
 * `rank` of every rank's gather buffer.  The buffers are allocated with rpl_peer_alloc (cudaMalloc +
 * cudaIpcGetMemHandle), the 64-byte handles are exchanged by the host (torch.distributed in this repo) and
 * opened with rpl_peer_open (cudaIpcOpenMemHandle: NVLink peer mapping).  Gather buffer layout:
 * [256-byte header: uint32 point count of every rank][world][slot_points][16 B]; size
 * rpl_peer_gather_bytes(world, slot_points).  peer_bases: HOST array [world] of device pointers, entry
 * `rank` = this rank's own buffer.  Completion: the stores are visible on the peers once this rank's
 * kernel has finished; a consumer needs one barrier over all ranks after the call (any tiny collective on
 * the same stream) and must not let the next push overwrite a buffer that is still being read
 * (rplidar_ros2_driver_b200/multi_gpu.py::PeerCloudGather alternates two buffers). */
#define RPL_IPC_HANDLE_BYTES 64u
#define RPL_MAX_PEERS 16u
size_t rpl_peer_gather_bytes(uint32_t world, uint32_t slot_points);
rpl_result rpl_peer_alloc(rpl_ctx* ctx, size_t bytes, void** dev_ptr, uint8_t* handle_out /* [64] */);
rpl_result rpl_peer_open(rpl_ctx* ctx, const uint8_t* handle /* [64] */, void** peer_ptr);
rpl_result rpl_peer_close(rpl_ctx* ctx, void* peer_ptr);
rpl_result rpl_peer_free(rpl_ctx* ctx, void* dev_ptr);
rpl_result rpl_cloud_fuse_push_dev(rpl_ctx* ctx, const float* xyzi, const uint32_t* point_counts, uint32_t n_scans,
                                   uint32_t stride, void* const* peer_bases, uint32_t world, uint32_t rank,
                                   uint32_t slot_points, uint32_t* offsets, uint32_t* total, void* stream);

/* ---- the exchange as a host-side C++ object (SURVEY.md 8(e): one process per GPU, ONE all-gather of the fused
 * cloud per step over NVLink, overlapped with the next batch's kernels) ------------------------------------
 * The reference has no analogue (it publishes one scan: src/rplidar_node.cpp:679); parity = every rank ends up
 * with the concatenation, in rank order, of what the ranks produce on their own.  NCCL is loaded at run time
 * (dlopen libnccl.so.2); the embedding process only carries the 128-byte unique id from rank 0 to the others.
 * rpl_exchange_create is collective (every rank, same id / world / slot_points); it creates the communicator
 * (ncclCommInitRank), a high-priority exchange stream, two gather buffers of `world` slots
 * [16-byte header: uint32 point count][slot_points x 16 B] and -- unless RPL_EXCHANGE_NO_PEER_MAP -- maps every
 * peer's buffers (CUDA IPC handles all-gathered through the communicator).
 * rpl_exchange_allgather packs the per-scan clouds of rpl_cloud_batch_dev (xyzi [n_scans][stride][4],
 * point_counts) into this rank's slot on `stream` and starts the transfer on the exchange stream:
 *   RPL_EXCHANGE_NCCL  one in-place ncclAllGather of the slot;
 *   RPL_EXCHANGE_COPY  world-1 peer-to-peer copies of the slot by the copy engines (no SM), then a 4-byte
 *                      all-reduce as the barrier.
 * `stream` is NOT made to wait for the transfer: the caller's next batch overlaps it.  *buffer_index (0/1) names
 * the buffer this step fills; a consumer calls rpl_exchange_wait(index, its stream) before reading the slots
 * (rpl_exchange_slot) and rpl_exchange_release(index, its stream) after its last read -- the exchange that reuses
 * the buffer two steps later waits for that.  A slot whose count exceeds slot_points overflowed (points dropped).
 * A step with n_scans == 0 (a rank with no streams, or none that closed a revolution) publishes an empty slot:
 * count 0; rpl_cloud_fuse_push_dev likewise writes 0 into header word `rank` of every peer. */
#define RPL_EXCHANGE_ID_BYTES 128u
#define RPL_EXCHANGE_NCCL 0u
#define RPL_EXCHANGE_COPY 1u
#define RPL_EXCHANGE_NO_PEER_MAP 1u /* create flag: NCCL mode only, no CUDA IPC mappings */
typedef struct rpl_exchange rpl_exchange;
rpl_result rpl_exchange_unique_id(uint8_t* id_out /* [128], call on rank 0 */);
rpl_result rpl_exchange_create(rpl_ctx* ctx, const uint8_t* id /* [128]; may be NULL when world == 1 */, uint32_t world,
                               uint32_t rank, uint32_t slot_points, uint32_t flags, rpl_exchange** out);
void rpl_exchange_destroy(rpl_exchange* ex); /* collective when world > 1 */
rpl_result rpl_exchange_allgather(rpl_exchange* ex, const float* xyzi, const uint32_t* point_counts, uint32_t n_scans,
                                  uint32_t stride, uint32_t mode, void* stream, uint32_t* buffer_index);
rpl_result rpl_exchange_wait(rpl_exchange* ex, uint32_t buffer_index, void* stream);
rpl_result rpl_exchange_release(rpl_exchange* ex, uint32_t buffer_index, void* stream);
rpl_result rpl_exchange_slot(rpl_exchange* ex, uint32_t buffer_index, uint32_t rank, const float** points,
                             const uint32_t** count);
rpl_result rpl_exchange_synchronize(rpl_exchange* ex);

/* ---- dense-capsule decode (SURVEY.md 8(f) rank 1: the step before the hot path) ------- */
/* Replaces UnpackerHandler_DenseCapsuleNode (reference
 * src/sdk/src/dataunpacker/unpacker/handler_capsules.cpp:639-791) for FRAMED capsules: answer
 * type 0x85, 84 bytes each (src/sdk/include/sl_lidar_cmd.h:223-234), one capsule per protocol
 * message.  capsules: [n_streams][stride_capsules][84]; nodes_out: [n_streams][stride_capsules*40]
 * HQ nodes in the order the reference's listener receives them; node_counts[s] = nodes decoded.
 * capsule_status (nullable): RPL_CAPSULE_* bits per capsule; capsule_node_offset (nullable):
 * nodes decoded before each capsule (so scan-reset / error events keep their place in the node
 * stream).  sync_state_in/out (nullable): the reference's function-static lastNodeSyncBit
 * entering / leaving every stream (0 = fresh process).  sample_duration_us:
 * SlamtecLidarTimingDesc::sample_duration_uS (sets the angular-jump discard threshold). */
#define RPL_DENSE_CAPSULE_BYTES 84u
#define RPL_CAPSULE_OK 1u                /* sync nibbles and checksum fine */
#define RPL_CAPSULE_SYNC 2u              /* first capsule of a revolution: scan reset requested */
#define RPL_CAPSULE_EMIT 4u              /* released the previous capsule's 40 nodes */
#define RPL_CAPSULE_DISCARD 8u           /* angular jump above the 100 Hz bound: nothing released */
#define RPL_CAPSULE_CHECKSUM_ERR 16u     /* ERR_EVENT_ON_EXP_CHECKSUM_ERR */
#define RPL_CAPSULE_ENCODER_RESET_ERR 32u /* ERR_EVENT_ON_EXP_ENCODER_RESET */
#define RPL_CAPSULE_BAD_FRAME 64u        /* wrong sync nibbles: outside the framed contract */
rpl_result rpl_decode_dense_batch_dev(rpl_ctx* ctx, const uint8_t* capsules, const uint32_t* capsule_counts,
                                      uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                      const uint32_t* sync_state_in, rpl_node_hq* nodes_out,
                                      uint32_t* node_counts, uint32_t* capsule_status,
                                      uint32_t* capsule_node_offset, uint32_t* sync_state_out, void* stream);
/* The same, and the decoder also lists where the revolutions start: scan_starts [n_streams][starts_stride] = node
 * offsets of the scan-start nodes of every stream (in no particular order), scan_start_counts[s] = how many there are
 * (more than starts_stride: the list is incomplete and must not be used).  rpl_assemble_scan_views_starts_dev takes
 * the list instead of reading every decoded node again. */
rpl_result rpl_decode_dense_batch_starts_dev(rpl_ctx* ctx, const uint8_t* capsules, const uint32_t* capsule_counts,
                                             uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                             const uint32_t* sync_state_in, rpl_node_hq* nodes_out,
                                             uint32_t* node_counts, uint32_t* capsule_status,
                                             uint32_t* capsule_node_offset, uint32_t* sync_state_out,
                                             uint32_t* scan_starts, uint32_t starts_stride, uint32_t* scan_start_counts,
                                             void* stream);
/* One stream, host buffers.  nodes_out must hold 40 * n_capsules nodes. */
rpl_result rpl_decode_dense(rpl_ctx* ctx, const uint8_t* capsules, uint32_t n_capsules,
                            uint32_t sample_duration_us, uint32_t* sync_state, rpl_node_hq* nodes_out,
                            uint32_t* node_count, uint32_t* capsule_status, uint32_t* capsule_node_offset);

/* ---- the other measurement answer formats (SURVEY.md 8(f) rank 1) ----------------------- */
/* ans_type is the SDK's answer type (reference src/sdk/include/sl_lidar_cmd.h:144-151):
 *   0x82 express capsules      84 B -> 32 nodes   UnpackerHandler_CapsuleNode           handler_capsules.cpp:109-266
 *   0x83 HQ capsules          781 B -> 96 nodes   UnpackerHandler_HQNode                handler_hqnode.cpp:93-172
 *   0x84 ultra capsules       132 B -> 96 nodes   UnpackerHandler_UltraCapsuleNode      handler_capsules.cpp:324-580
 *   0x85 dense capsules        84 B -> 40 nodes   (same kernel as rpl_decode_dense_batch_dev)
 *   0x86 ultra-dense capsules 170 B -> 64 nodes   UnpackerHandler_UltraDenseCapsuleNode handler_capsules.cpp:852-1047
 * (reference src/sdk/src/dataunpacker/unpacker/).  Framed input as for the dense decoder:
 * capsules [n_streams][stride_capsules][rpl_capsule_bytes(ans_type)], nodes_out
 * [n_streams][stride_capsules * rpl_capsule_nodes(ans_type)].  state_in / state_out (nullable):
 * [n_streams][2] = {scan-start flag of the last node, last distance} -- the decoder state the SDK
 * keeps across capsules for the dense (word 0) and ultra-dense (both) formats; 0 on a fresh decoder.
 * The per-capsule status words are the RPL_CAPSULE_* bits above. */
/* sl::SlamtecLidarTimingDesc (reference src/sdk/include/sl_lidar_driver.h:156-166). */
typedef struct rpl_timing {
  uint32_t sample_duration_us;
  uint32_t native_baudrate;        /* 0 = the per-format default the SDK assumes */
  uint32_t linkage_delay_us;
  uint32_t native_interface_type;  /* sl::LIDARInterfaceType: 0 UART, 1 ETHERNET, 2 USB, 5 CANBUS */
} rpl_timing;
#define RPL_ANS_MEASUREMENT 0x81u
#define RPL_ANS_MEASUREMENT_CAPSULED 0x82u
#define RPL_ANS_MEASUREMENT_HQ 0x83u
#define RPL_ANS_MEASUREMENT_CAPSULED_ULTRA 0x84u
#define RPL_ANS_MEASUREMENT_DENSE_CAPSULED 0x85u
#define RPL_ANS_MEASUREMENT_ULTRA_DENSE_CAPSULED 0x86u
uint32_t rpl_capsule_bytes(uint32_t ans_type); /* 0 for an unknown type */
uint32_t rpl_capsule_nodes(uint32_t ans_type);
rpl_result rpl_decode_capsules_batch_dev(rpl_ctx* ctx, uint32_t ans_type, const uint8_t* capsules,
                                         const uint32_t* capsule_counts, uint32_t n_streams,
                                         uint32_t stride_capsules, uint32_t sample_duration_us,
                                         const uint32_t* state_in, rpl_node_hq* nodes_out, uint32_t* node_counts,
                                         uint32_t* capsule_status, uint32_t* capsule_node_offset,
                                         uint32_t* state_out, void* stream);
/* One stream, host buffers.  state: in/out [2] (nullable).  timing / capsule_rx_us / node_ts_us (nullable
 * together): also return the per-node stamps of rpl_node_timestamps_dev (below) for the receive times
 * capsule_rx_us[n_capsules]; sample_duration_us is then taken from timing. */
rpl_result rpl_decode_capsules(rpl_ctx* ctx, uint32_t ans_type, const uint8_t* capsules, uint32_t n_capsules,
                               uint32_t sample_duration_us, uint32_t* state, rpl_node_hq* nodes_out,
                               uint32_t* node_count, uint32_t* capsule_status, uint32_t* capsule_node_offset,
                               const rpl_timing* timing, const uint64_t* capsule_rx_us, uint64_t* node_ts_us);
/* Byte-level framing of RAW capsule streams (0x82, 0x84, 0x85, 0x86) with the SDK's resynchronisation: the hunt for
 * the two sync nibbles of UnpackerHandler_{Capsule,UltraCapsule,DenseCapsule,UltraDenseCapsule}Node::onData
 * (reference src/sdk/src/dataunpacker/unpacker/handler_capsules.cpp:107-135, 324-353, 639-668, 852-880).
 * bytes [n_streams][stride_bytes] -> capsules_out [n_streams][stride_capsules][rpl_capsule_bytes(ans_type)], the
 * input of the decoders above; every stretch of bytes the SDK would skip becomes ONE all-zero capsule (decoded as
 * RPL_CAPSULE_BAD_FRAME: the decoders then forget the previous capsule, as the SDK does).  capsule_counts_out[s] >
 * stride_capsules means the output overflowed (a stream of B bytes needs at most 2 * (B / frame size) + 2 slots);
 * bytes_left_out (nullable): bytes of an unfinished frame at the end of the stream -- prepend them to the next
 * piece of the stream. */
rpl_result rpl_frame_capsules_dev(rpl_ctx* ctx, uint32_t ans_type, const uint8_t* bytes, const uint32_t* byte_counts,
                                  uint32_t n_streams, uint32_t stride_bytes, uint8_t* capsules_out,
                                  uint32_t stride_capsules, uint32_t* capsule_counts_out, uint32_t* bytes_left_out,
                                  void* stream);
/* 0x81 standard measurement nodes (5 bytes each) from RAW byte streams, with the byte-level
 * resynchronisation of UnpackerHandler_NormalNode::onData (handler_normalnode.cpp:88-141): exact on
 * misframed / corrupted streams.  bytes [n_streams][stride_bytes]; nodes_out
 * [n_streams][stride_bytes / 5]; fsm_state_out (nullable): bytes still buffered at the end; node_end
 * (nullable, [n_streams][stride_bytes / 5]): index of the last byte of each decoded record (what
 * rpl_normal_timestamps_dev needs to find the piece of the stream a record arrived in). */
rpl_result rpl_decode_normal_batch_dev(rpl_ctx* ctx, const uint8_t* bytes, const uint32_t* byte_counts,
                                       uint32_t n_streams, uint32_t stride_bytes, rpl_node_hq* nodes_out,
                                       uint32_t* node_counts, uint32_t* fsm_state_out, uint32_t* node_end,
                                       void* stream);
rpl_result rpl_decode_normal(rpl_ctx* ctx, const uint8_t* bytes, uint32_t n_bytes, rpl_node_hq* nodes_out,
                             uint32_t* node_count);

/* ---- scan assembly (SURVEY.md 8(f) rank 2: node stream -> scans, on the device) -------- */
/* Replaces ScanDataHolder::pushScanNodeData / rewindCurrentScanData (reference
 * src/sdk/src/sl_lidar_driver.cpp:272-315).  nodes: [n_streams][stride_nodes] decoded streams
 * (rpl_decode_dense_batch_dev output).  capsule_status / capsule_node_offset / capsule_counts
 * (nullable together): the decoder's per-capsule report, from which the scan-reset requests are
 * taken (one before every RPL_CAPSULE_SYNC capsule).  max_nodes: holder capacity (8192 in the SDK);
 * scan_stride >= max_nodes.  scans_out: [n_streams][max_scans][scan_stride]; scan_len:
 * [n_streams][max_scans]; scans_per_stream[s] = scans published (only the first max_scans stored).
 * The output is laid out as the input of rpl_scan_batch_dev (n_scans = n_streams * max_scans with
 * scan_len as counts; unused slots must be zeroed by the caller or have length 0).
 * node_ts_us (nullable, [n_streams][stride_nodes]) / scan_begin_ts_us (nullable,
 * [n_streams][max_scans]): every published scan reports the stamp of the scan-start node that opened
 * it (ScanDataHolder::_scan_begin_timestamp_uS, :293,:326-328; what grabScanDataHqWithTimeStamp returns). */
rpl_result rpl_assemble_scans_dev(rpl_ctx* ctx, const rpl_node_hq* nodes, const uint32_t* node_counts,
                                  uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                  const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                  uint32_t stride_capsules, uint32_t max_nodes, uint32_t max_scans,
                                  uint32_t scan_stride, rpl_node_hq* scans_out, uint32_t* scan_len,
                                  uint32_t* scans_per_stream, const uint64_t* node_ts_us,
                                  uint64_t* scan_begin_ts_us, void* stream);

/* The same cut WITHOUT the copy: a published scan is returned as a view {first node, count} into the node buffer
 * itself (first counts from the start of `nodes`, across streams), and rpl_scan_views_dev reads the revolutions
 * where the decoder left them -- the capsule -> LaserScan chain then moves every node through HBM once less in
 * each direction.  views_out / scan_len: [n_streams][max_scans], unused entries are {0, 0}.  The holder's capacity
 * rule (a scan longer than max_nodes keeps overwriting its last entry) is applied IN PLACE: node first+max_nodes-1
 * of such a scan is overwritten with the scan's last node (the nodes behind it are dropped either way), which is
 * why `nodes` is not const here. */
typedef struct rpl_scan_view {
  uint32_t first; /* index of the scan's first node in the whole node buffer */
  uint32_t count;
} rpl_scan_view;
rpl_result rpl_assemble_scan_views_dev(rpl_ctx* ctx, rpl_node_hq* nodes, const uint32_t* node_counts,
                                       uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                       const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                       uint32_t stride_capsules, uint32_t max_nodes, uint32_t max_scans,
                                       rpl_scan_view* views_out, uint32_t* scan_len, uint32_t* scans_per_stream,
                                       const uint64_t* node_ts_us, uint64_t* scan_begin_ts_us, void* stream);
/* rpl_assemble_scan_views_dev with the decoder's scan-start list (rpl_decode_dense_batch_starts_dev): a stream whose
 * list is complete is cut without touching its nodes; one whose list overflowed falls back to reading them. */
rpl_result rpl_assemble_scan_views_starts_dev(rpl_ctx* ctx, rpl_node_hq* nodes, const uint32_t* node_counts,
                                              uint32_t n_streams, uint32_t stride_nodes, const uint32_t* capsule_status,
                                              const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                              uint32_t stride_capsules, const uint32_t* scan_starts,
                                              uint32_t starts_stride, const uint32_t* scan_start_counts,
                                              uint32_t max_nodes, uint32_t max_scans, rpl_scan_view* views_out,
                                              uint32_t* scan_len, uint32_t* scans_per_stream, const uint64_t* node_ts_us,
                                              uint64_t* scan_begin_ts_us, void* stream);
/* rpl_scan_batch_dev over views: scan s = views[s].count nodes from nodes[views[s].first]; nodes_total = nodes in
 * the buffer; outputs laid out [n_scans][stride] as before (stride >= every count, stride <= 8192: the views are
 * served by the shared-memory kernels).  `nodes` must be 16-byte aligned. */
rpl_result rpl_scan_views_dev(rpl_ctx* ctx, const rpl_node_hq* nodes, uint64_t nodes_total, const rpl_scan_view* views,
                              uint32_t n_scans, uint32_t stride, const rpl_scan_params* params, rpl_node_hq* nodes_out,
                              float* ranges, float* intensities, uint32_t* beam_counts, float* angle_increment,
                              uint32_t* status, uint32_t* path, void* stream);

/* Wire bytes -> LaserScan in ONE host call: framed dense (0x85) capsules in host memory -> H2D -> decode ->
 * scan views -> scan kernel -> D2H, chunked over the two lanes so that copies and kernels overlap.  Per stream this is
 * the reference's whole data path after the protocol codec: UnpackerHandler_DenseCapsuleNode::onData
 * (src/sdk/src/dataunpacker/unpacker/handler_capsules.cpp:639-791) -> ScanDataHolder::pushScanNodeData
 * (src/sdk/src/sl_lidar_driver.cpp:272-315) -> grab_scan_data with ascendScanData (src/lidar_driver_wrapper.cpp:307-342,
 * src/sdk/src/sl_lidar_driver.cpp:128-184) -> publish_scan (src/rplidar_node.cpp:556-680).  2.1 bytes per
 * point cross the host link on the way in instead of the 8 of a decoded node.  capsules: host
 * [n_streams][stride_capsules][84]; outputs: host ranges / intensities [n_streams * max_scans][max_nodes],
 * beam_counts / angle_increment (nullable) [n_streams * max_scans] (slot k of stream s at s * max_scans + k; unused
 * slots have beam count 0), scans_per_stream [n_streams].  max_nodes: even, <= 8192, at least the longest
 * revolution (longer ones are cut by the holder's capacity rule); the context's max_scans must cover
 * max_scans of at least one stream.  Pinned host memory (rpl_host_alloc) keeps the copies asynchronous. */
rpl_result rpl_chain_dense_laserscan(rpl_ctx* ctx, const uint8_t* capsules, const uint32_t* capsule_counts,
                                     uint32_t n_streams, uint32_t stride_capsules, uint32_t sample_duration_us,
                                     const rpl_scan_params* params, uint32_t max_nodes, uint32_t max_scans,
                                     float* ranges, float* intensities, uint32_t* beam_counts, float* angle_increment,
                                     uint32_t* scans_per_stream);

/* Capsule stream session: decode -> assemble -> LaserScan for live streams of one capsule answer type.  The stateless
 * calls (rpl_chain_dense_laserscan; rpl_decode_capsules_batch_dev -> rpl_assemble_scan_views_dev -> rpl_scan_views_dev)
 * treat every call as a whole recording: the last capsule, which the express, ultra, dense and ultra-dense unpackers
 * hold until the next one arrives, and the revolution still open at the end are lost.  A session keeps both per stream
 * on the device, so that for ANY split of a stream's capsules into pushes the scans published over the pushes, in
 * order, are the scans of the whole stream (the SDK's unpacker and ScanDataHolder fed the same bytes).  A scan is
 * published by the push that delivers the scan-start node closing it -- with the held capsule, possibly one push after
 * its capsule.  A stream with 0 capsules in a push keeps its state and publishes nothing.  The first push of a fresh
 * session publishes what the stateless device path does on the same capsules (dense: what rpl_chain_dense_laserscan
 * does).
 *   create:  ans_type 0x82 express, 0x83 HQ, 0x84 ultra, 0x85 dense or 0x86 ultra-dense (0x81 standard nodes, which
 *            come in no capsules: rpl_capsule_stream_create_bytes; anything else: RPL_RESULT_INVALID_DATA); n_streams,
 *            stride_capsules (most capsules per stream in one push), max_nodes
 *            (even, <= 8192: the holder capacity and the output row), max_scans (slots per stream per push); the
 *            context's max_scans must cover one stream's max_scans.  The session borrows the context (its lanes, whose
 *            staging memory a host push grows to what it needs, and the assembler scratch) and is destroyed before
 *            it.  Device memory of its own: two node arenas of
 *            n_streams * (max_nodes + rpl_capsule_nodes(ans_type) * stride_capsules) nodes each (DESIGN.md 5.7), which
 *            must stay below 2^32 nodes, plus per-capsule reports.
 *   push:    host buffers, synchronous, chunked (about 16 MiB of capsules) over the context's two lanes: capsules
 *            [n_streams][stride_capsules][rpl_capsule_bytes(ans_type)], capsule_counts [n_streams] (<= stride_capsules),
 *            outputs [n_streams * max_scans][max_nodes] / [n_streams * max_scans] (slot k of stream s = the k-th scan
 *            this push published for s), scans_per_stream [n_streams] (> max_scans: scans were dropped).  Dense capsule
 *            buffers must be 4-byte aligned, as for rpl_decode_capsules_batch_dev.
 *   push_dev: the same on device buffers, asynchronous on `stream` (NULL = the context's stream).  Counts above the
 *            stride are clamped to it.
 *   reset:   the SDK's unpacker reset + holder reset (a reconnect): drop the held capsule, the decoder's scan-start
 *            flag and smoothed last distance, and the open revolution of every stream whose stream_mask entry is
 *            non-zero (NULL = all).
 *   state:   synchronous; open_nodes [n_streams] = nodes in each stream's open revolution (capped at max_nodes),
 *            held_capsule [n_streams] = 1 when a valid capsule is held for the next push (always 0 for HQ and 0x81,
 *            which hold none), held_bytes [n_streams] = the bytes a byte session holds for the next push (always 0 on a
 *            framed session); every pointer nullable.
 *   push_ts / push_ts_dev: a stamped push.  push / push_dev with the receive time of every capsule, capsule_rx_us
 *            [n_streams][stride_capsules] (the time of the read that delivered the capsule's last byte, when the
 *            SDK's unpacker calls getCurrentTimestamp_uS), and the timing of rpl_node_timestamps_dev, whose
 *            sample_duration_us the decoder takes.  Also returns scan_begin_ts_us [n_streams * max_scans] (slots as
 *            beam_counts, unused ones 0): the stamp of the scan-start node that opened each published scan, the
 *            holder's _scan_begin_timestamp_uS (sl_lidar_driver.cpp:293).  For any split into pushes the stamps
 *            published over the pushes, in order, are those of the whole stream (rpl_node_timestamps_dev ->
 *            rpl_assemble_scans_dev on the concatenation).  A scan opened pushes ago keeps its stamp; for express and
 *            ultra, a scan-start node in a capsule held over a push counts from the held capsule's receive time.
 *            Stamped and unstamped pushes mix on one session (an unstamped push runs exactly the unstamped kernels and
 *            keeps no stamp), so a stamp that depends on a receive time the session was not given or did not keep is
 *            reported as 0: a scan opened in an unstamped push or still open across one, or (express, ultra) opened
 *            by a node of a capsule an unstamped push held.  Null timing, receive times or scan_begin_ts_us, or 8-byte
 *            buffers not 8-byte aligned: RPL_RESULT_INVALID_DATA. */
typedef struct rpl_capsule_stream rpl_capsule_stream;
rpl_result rpl_capsule_stream_create(rpl_ctx* ctx, uint32_t ans_type, uint32_t n_streams, uint32_t stride_capsules,
                                     uint32_t max_nodes, uint32_t max_scans, rpl_capsule_stream** out);
void rpl_capsule_stream_destroy(rpl_capsule_stream* s);
rpl_result rpl_capsule_stream_push(rpl_capsule_stream* s, const uint8_t* capsules, const uint32_t* capsule_counts,
                                   uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                   float* intensities, uint32_t* beam_counts, float* angle_increment,
                                   uint32_t* scans_per_stream);
rpl_result rpl_capsule_stream_push_dev(rpl_capsule_stream* s, const uint8_t* capsules, const uint32_t* capsule_counts,
                                       uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                       float* intensities, uint32_t* beam_counts, float* angle_increment,
                                       uint32_t* scans_per_stream, void* stream);
rpl_result rpl_capsule_stream_push_ts(rpl_capsule_stream* s, const uint8_t* capsules, const uint32_t* capsule_counts,
                                      const rpl_timing* timing, const uint64_t* capsule_rx_us,
                                      const rpl_scan_params* params, float* ranges, float* intensities,
                                      uint32_t* beam_counts, float* angle_increment, uint32_t* scans_per_stream,
                                      uint64_t* scan_begin_ts_us);
rpl_result rpl_capsule_stream_push_ts_dev(rpl_capsule_stream* s, const uint8_t* capsules,
                                          const uint32_t* capsule_counts, const rpl_timing* timing,
                                          const uint64_t* capsule_rx_us, const rpl_scan_params* params, float* ranges,
                                          float* intensities, uint32_t* beam_counts, float* angle_increment,
                                          uint32_t* scans_per_stream, uint64_t* scan_begin_ts_us, void* stream);
rpl_result rpl_capsule_stream_reset(rpl_capsule_stream* s, const uint8_t* stream_mask);
rpl_result rpl_capsule_stream_state(rpl_capsule_stream* s, uint32_t* open_nodes, uint32_t* held_capsule,
                                    uint32_t* held_bytes);

/* Session counters: per stream, what the session decoded and what it had to throw away, accumulated on the device by
 * the kernels every push already runs, from create on, over every push flavour (framed or bytes, host or _dev, stamped
 * or not, with or without RPL_FLAG_PER_STREAM).  Every counter but scans_unreturned depends on the stream alone, not on
 * how it is split into pushes: after any split it equals what one push of the whole stream counts, and what the SDK's
 * unpacker and ScanDataHolder fed the same bytes in any pieces count.  An event is counted by the push whose input
 * completes it (a discard: by the capsule that would have released the held one; an overwrite: by the node that
 * overwrites).  A stream with a count of 0 in a push changes no counter; a push that returns an error may have counted
 * part of its input.  rpl_capsule_stream_reset leaves the counters alone (a reconnect is not a new lidar); the bytes it
 * drops from a held frame are counted nowhere.  On a byte session never reset, with held_bytes of
 * rpl_capsule_stream_state: bytes_in == frames * frame size + skipped_bytes + held_bytes (0x81: 5 * frames + ...).
 * References: src/sdk/src/dataunpacker/unpacker/handler_capsules.cpp (express :112-136,:170,:185; ultra :387,:402;
 * dense :703,:717; ultra-dense :915,:929), handler_hqnode.cpp:95-172, handler_normalnode.cpp:92-113,
 * dataunpacker.cpp:199-202, sl_lidar_driver.cpp:272-315 (ScanDataHolder), :1645-1653. */
typedef struct rpl_stream_counters {
  uint64_t bytes_in;           /* bytes taken from the caller's buffers (_dev: after the clamp); a framed session:
                                  capsules x capsule size */
  uint64_t frames;             /* frames the sync hunt completed (byte sessions), capsules pushed (framed sessions),
                                  records decoded (0x81) */
  uint64_t skipped_bytes;      /* bytes the unpacker's sync hunt skipped (handler_capsules.cpp:112-136 and siblings,
                                  handler_hqnode.cpp:95-172, handler_normalnode.cpp:92-113), a first sync byte dropped
                                  with a second that does not match included; 0 on a framed session */
  uint64_t bad_frames;         /* capsules decoded as RPL_CAPSULE_BAD_FRAME: a byte session's all-zero capsule per run
                                  of skipped bytes, a framed session's capsules with wrong sync nibbles; 0 on 0x81 */
  uint64_t checksum_errors;    /* ERR_EVENT_ON_EXP_CHECKSUM_ERR (dataunpacker.h:52-65; HQ: CRC, handler_hqnode.cpp:162) */
  uint64_t encoder_resets;     /* ERR_EVENT_ON_EXP_ENCODER_RESET (dataunpacker.h:52-65) */
  uint64_t scan_resets;        /* onHQNodeScanResetReq calls (dataunpacker.cpp:199-202) */
  uint64_t discarded_capsules; /* capsules whose nodes the angular-jump bound kept back (RPL_CAPSULE_DISCARD), under the
                                  stream's own sample duration with RPL_FLAG_PER_STREAM */
  uint64_t nodes;              /* onHQNodeDecoded calls (sl_lidar_driver.cpp:1645-1649) */
  uint64_t nodes_unopened;     /* nodes the holder dropped because no scan was open (sl_lidar_driver.cpp:296-298) */
  uint64_t nodes_overwritten;  /* nodes that replaced the last entry of a revolution longer than the session's max_nodes
                                  (sl_lidar_driver.cpp:302-305) */
  uint64_t scans_rewound;      /* scan resets that emptied a non-empty revolution in progress (sl_lidar_driver.cpp:312-315) */
  uint64_t scans_published;    /* scans the holder completed (sl_lidar_driver.cpp:279-288) */
  uint64_t scans_unreturned;   /* published scans a push could not return, beyond its max_scans (the sum over pushes of
                                  scans_per_stream - max_scans where positive) */
} rpl_stream_counters;
/* Synchronous: waits for every push issued before it, on any CUDA stream, copies the n_streams records to out
 * (nullable: no copy), then zeroes the records of the streams whose clear_mask entry is non-zero (nullable: none)
 * before any later push runs.  Null session: RPL_RESULT_INVALID_DATA. */
rpl_result rpl_capsule_stream_counters(rpl_capsule_stream* s, rpl_stream_counters* out /* [n_streams] */,
                                       const uint8_t* clear_mask /* [n_streams] */);

/* Byte session: the session fed the RAW serial stream after the answer descriptor, any number of bytes per push, a
 * push ending anywhere -- what the SDK's protocol codec hands LIDARSampleDataUnpacker::onSampleData.  Per stream the
 * device also keeps the unpacker's state between frames, so for ANY split of a stream's bytes into pushes the scans
 * (and, stamped, their scan-begin stamps) published over the pushes are those of the SDK's unpacker and ScanDataHolder
 * fed the whole stream.
 *   Capsule answer types (0x82..0x86): the device keeps the unpacker's search for the sync bytes
 *            (handler_capsules.cpp:107-135 express, :324-353 ultra, :639-668 dense, :852-880 ultra-dense;
 *            handler_hqnode.cpp:95-172 HQ): the search position, the bytes of the unfinished frame (up to the frame
 *            size - 1) and whether bytes were skipped since the last frame (which clears the handler's
 *            _is_previous_capsuledataRdy).  The split may fall between the two sync bytes, inside a frame or inside a
 *            run of skipped bytes.  Each push is framed on the device (rpl_frame_capsules_dev's framing carried across
 *            pushes; HQ: a byte other than 0xA5 is skipped while waiting, a 0xA5 and the 780 bytes behind it are a
 *            frame) and then decoded as a framed push of those capsules.
 *   0x81 standard nodes (the SDK's "Standard" scan mode, the only mode of the legacy A-series lidars): the device
 *            keeps the unpacker's 0..4 bytes of an unfinished record; the split may fall through a record, a
 *            resynchronisation or a scan-start record (UnpackerHandler_NormalNode).  There is no framing and no framer
 *            record: the held record's byte machine is the framing.  The standard unpacker requests no scan resets and
 *            its decoder takes no sample duration (sample_duration_us is ignored).  The first push of a fresh session
 *            publishes what rpl_decode_normal_batch_dev -> rpl_assemble_scan_views_dev -> rpl_scan_views_dev does on
 *            the same bytes.
 *   create_bytes: ans_type 0x81..0x86 (anything else RPL_RESULT_INVALID_DATA), stride_bytes (most bytes per stream in
 *            one push), max_nodes, max_scans: the rules of rpl_capsule_stream_create.  The session's own device memory:
 *            capsule answer types, with F = ceil(stride_bytes / frame size) (the frames a push can complete) and
 *            S = 2 * F capsule slots (F for HQ: every frame can follow a run of skipped bytes, reported as one all-zero
 *            capsule), two node arenas of n_streams * (max_nodes + rpl_capsule_nodes(ans_type) * F) nodes of 8 bytes,
 *            n_streams * S * (frame size + 16) bytes of framed capsules, their reports and receive times, and an
 *            800-byte framer record per stream; 0x81, two node arenas of n_streams * (max_nodes + (stride_bytes + 4) /
 *            5 rounded up to even) nodes.  Either way the arenas must stay below 2^32 nodes.
 *   push_bytes / push_bytes_dev: bytes [n_streams][stride_bytes] (any alignment), byte_counts [n_streams] (<= stride_bytes;
 *            _dev: counts above it clamped), sample_duration_us and outputs as for rpl_capsule_stream_push.
 *   push_bytes_ts / push_bytes_ts_dev: a stamped push, as rpl_capsule_stream_push_ts: chunk_rx_us [n_streams][ceil(
 *            stride_bytes / chunk_bytes)], chunk c the receive time of bytes [c * chunk_bytes, (c + 1) * chunk_bytes) of
 *            THIS push (the rule of rpl_normal_timestamps_dev); a capsule or record gets the time of the chunk holding
 *            its last byte (when the handler completes it), also when it began in an earlier push.  chunk_bytes == 0:
 *            RPL_RESULT_INVALID_DATA.
 *   reset:   rpl_capsule_stream_reset, which on a byte session also restarts the search (the handlers' reset();
 *            0x81: _cached_scan_node_buf_pos = 0).
 *   state:   rpl_capsule_stream_state; held_bytes = bytes of the unfinished frame (0..frame size - 1), 0x81 of the
 *            unfinished record (0..4), held for the next push.  held_capsule is 0 while skipped bytes wait to be
 *            reported.
 * A framed push (rpl_capsule_stream_push*) on a byte session, or a byte push on a framed session: RPL_RESULT_INVALID_DATA. */
rpl_result rpl_capsule_stream_create_bytes(rpl_ctx* ctx, uint32_t ans_type, uint32_t n_streams, uint32_t stride_bytes,
                                           uint32_t max_nodes, uint32_t max_scans, rpl_capsule_stream** out);
rpl_result rpl_capsule_stream_push_bytes(rpl_capsule_stream* s, const uint8_t* bytes, const uint32_t* byte_counts,
                                         uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                         float* intensities, uint32_t* beam_counts, float* angle_increment,
                                         uint32_t* scans_per_stream);
rpl_result rpl_capsule_stream_push_bytes_dev(rpl_capsule_stream* s, const uint8_t* bytes, const uint32_t* byte_counts,
                                             uint32_t sample_duration_us, const rpl_scan_params* params, float* ranges,
                                             float* intensities, uint32_t* beam_counts, float* angle_increment,
                                             uint32_t* scans_per_stream, void* stream);
rpl_result rpl_capsule_stream_push_bytes_ts(rpl_capsule_stream* s, const uint8_t* bytes, const uint32_t* byte_counts,
                                            const rpl_timing* timing, uint32_t chunk_bytes, const uint64_t* chunk_rx_us,
                                            const rpl_scan_params* params, float* ranges, float* intensities,
                                            uint32_t* beam_counts, float* angle_increment, uint32_t* scans_per_stream,
                                            uint64_t* scan_begin_ts_us);
rpl_result rpl_capsule_stream_push_bytes_ts_dev(rpl_capsule_stream* s, const uint8_t* bytes,
                                                const uint32_t* byte_counts, const rpl_timing* timing,
                                                uint32_t chunk_bytes, const uint64_t* chunk_rx_us,
                                                const rpl_scan_params* params, float* ranges, float* intensities,
                                                uint32_t* beam_counts, float* angle_increment,
                                                uint32_t* scans_per_stream, uint64_t* scan_begin_ts_us, void* stream);
/* Mixed byte sessions: a byte session in which every stream has its own answer type, and a stream's type can change
 * between pushes, as the node's scan_mode parameter restarts the scan in another mode (rplidar_node.cpp:737-767).
 *   create_bytes_mixed: ans_types [n_streams] (host), each 0x81..0x86; stride_bytes, max_nodes, max_scans and the 2^32
 *            node limit as for create_bytes.  Every stream's regions are sized for the largest of the six types, so
 *            that any later switch fits without reallocating: with F(t) = ceil(stride_bytes / frame size of t) and
 *            S(t) = 2 * F(t) capsule slots (F for HQ), two node arenas of n_streams * (max_nodes + 96 *
 *            ceil(stride_bytes / 132)) nodes of 8 bytes (ultra completes the most nodes from a push), n_streams *
 *            max_t(S(t) * frame size of t) bytes of framed capsules (rounded up to 16) and n_streams * S(0x82) reports
 *            and receive times of 16 bytes, an 800-byte framer record, the 0x81 scan-end table of n_streams * (arena
 *            stride - max_nodes) words and the dense scan-start list.  A null ans_types, a type outside 0x81..0x86 or
 *            framed capsules of 2^32 bytes or more per stream (stride_bytes near 2^31): RPL_RESULT_INVALID_DATA.
 *   set_answer_types: the masked streams (stream_mask nullable: all) take ans_types[s]; synchronous, it waits for the
 *            session's device calls in flight.  A stream whose type changes is reset exactly as rpl_capsule_stream_reset
 *            resets it (held frame and search, held record, open revolution and its stamp, held receive time: the
 *            SDK's startScan* holder reset and unpacker enable, sl_lidar_driver.cpp:640-657) and decodes as the new
 *            type from the next push on; a stream whose type does not change is left alone (the node skips an
 *            unchanged scan_mode, :741-743).  Counters, lidar and frame settings are kept, and the last push's clouds,
 *            nodes and messages do not change.  A null ans_types, a masked type outside 0x81..0x86 or a session not
 *            made by create_bytes_mixed: RPL_RESULT_INVALID_DATA and no stream changes.
 *   Every byte session call (push_bytes*, with or without RPL_FLAG_PER_STREAM, reset, state, counters, set_frames,
 *            set_lidars, cloud*, nodes*, laserscan_msgs*, cloud_msgs*) takes a mixed session; state reports held_bytes
 *            and held_capsule by each stream's own type.  Without RPL_FLAG_PER_STREAM a push's sample_duration_us
 *            serves every capsule-type stream and is ignored for 0x81 streams (a session of 0x81 streams alone
 *            checks none).  Framed pushes: RPL_RESULT_INVALID_DATA, as on any byte session.
 *   Definition: for any split into pushes, stream s gives bit for bit what a one-stream create_bytes session of its
 *            type gives when fed the same pieces with the same params, in every output of every call above.  Across a
 *            switch the stream's outputs are two such sessions in a row: the old type's up to the switch, then a fresh
 *            session of the new type fed only the bytes after it; its counters are the sum of the two sessions'.
 *   Cost: each push runs the framer (capsule types), decoder and assembler once per answer type present in each
 *            chunk, over that type's streams, and the scan kernels once per chunk. */
rpl_result rpl_capsule_stream_create_bytes_mixed(rpl_ctx* ctx, const uint32_t* ans_types, uint32_t n_streams,
                                                 uint32_t stride_bytes, uint32_t max_nodes, uint32_t max_scans,
                                                 rpl_capsule_stream** out);
rpl_result rpl_capsule_stream_set_answer_types(rpl_capsule_stream* s, const uint32_t* ans_types,
                                               const uint8_t* stream_mask);
/* Session clouds: the PointCloud2 chain of rpl_cloud_batch_dev over the scans the session's last successful push
 * published, read in place from the session's node arenas (no copy of the scans, no second decode).
 *   Which scans: xyzi [n_streams * max_scans][max_nodes][4] floats (the layout of rpl_cloud_batch_dev), point_counts
 *            [n_streams * max_scans]; slot k of stream s is the scan whose LaserScan (and scan-begin stamp) that push
 *            wrote to slot k of stream s; unused slots get point count 0 (their rows are not written).
 *   Definition: each cloud is bit for bit what rpl_cloud_batch_dev returns with the same params for that scan's nodes,
 *            the holder's scan after its capacity rule (the ascended buffer does not matter: the cloud drops
 *            unmeasured nodes).  Flags 0 fuses SOR / voxel grid into the shared-memory kernel whenever the voxel rule
 *            of rpl_cloud_batch_dev allows it, also for max_nodes above 4096 (a revolution longer than 4096 nodes then
 *            takes the general kernel and the separate passes); RPL_CLOUD_NO_FUSED runs them as separate passes.
 *   Every push flavour: framed or byte pushes, host or device, stamped or not (a byte session: the
 *            rpl_capsule_stream_* pair).  The clouds can be taken any number of times between that push and the
 *            next; a reset in between does not change them.  Before any push, after a push that failed, with
 *            sor_k > 32, outside the voxel rule of rpl_cloud_batch_dev or with a null pointer:
 *            RPL_RESULT_INVALID_DATA.
 *   cloud_dev: device buffers, asynchronous on `stream` (NULL = the context's stream).  It waits for the session's
 *            last push (on any stream) and the session's next push waits for it.  Its scan kernels and SOR / voxel
 *            passes take turns with every other call of the context on its scan scratch, whatever their stream.
 *   cloud:   host buffers, synchronous, chunked over the context's lanes as a host push is. */
rpl_result rpl_capsule_stream_cloud_dev(rpl_capsule_stream* s, const rpl_cloud_params* params, float* xyzi,
                                        uint32_t* point_counts, void* stream);
rpl_result rpl_capsule_stream_cloud(rpl_capsule_stream* s, const rpl_cloud_params* params, float* xyzi,
                                    uint32_t* point_counts);

/* Session nodes: the node buffer RealLidarDriver::grab_scan_data returns (src/lidar_driver_wrapper.cpp:307-342) for
 * every scan the session's last successful push published -- the holder's scan, run through ascendScanData when
 * angle_compensate is set (:326-329, return value ignored) -- packed one behind the other.
 *   Which scans, repeat calls, ordering and errors: those of the session clouds above.  Slot i = s * max_scans + k is
 *            the scan whose LaserScan and scan-begin stamp that push wrote to slot k of stream s.  Every push flavour;
 *            callable any number of times between that push and the next, a reset in between changes nothing.  Before
 *            any push, after a push that failed, or with a null nodes, node_offsets, node_counts, status or
 *            total_nodes: RPL_RESULT_INVALID_DATA.
 *   Definition: with H the holder's scan (the view's nodes after the assembler's capacity rule), node_counts[i] =
 *            len(H), 0 for an unused slot.  Where ascend applies to the stream, the buffer is ascendScanData(H) under
 *            this library's tie rule (equal final keys keep buffer order): bit for bit what rpl_scan_batch_dev writes
 *            to nodes_out for H with apply_ascend = 1, and on tie-free revolutions the SDK's own result.  status[i] is
 *            the SDK's return value: RPL_RESULT_OK, or RPL_RESULT_OPERATION_FAIL when H has no measured node, the
 *            buffer then being H unchanged (src/sdk/src/sl_lidar_driver.cpp:150-151; the wrapper still returns the
 *            nodes).  Where ascend does not apply, the buffer is H unchanged and the status RPL_RESULT_OK.  A slot
 *            without a buffer (unused, or every slot when the buffers do not fit) has status RPL_RESULT_OK.
 *   Which streams are ascended: ascend_per_stream == NULL: every stream iff apply_ascend != 0.  Otherwise stream s iff
 *            ascend_per_stream[s] != 0 ([n_streams], host memory in both forms), and apply_ascend is ignored:
 *            angle_compensate is a parameter of each node in the reference (connect(port, baud,
 *            use_geometric_compensation)).  rpl_lidar_settings.pad plays no part.
 *   Packing: buffer i starts at nodes + node_offsets[i]; node_offsets [n_streams * max_scans] is the exclusive scan, in
 *            slot order, of the counts each rounded up to even, so every buffer is 16-byte aligned when nodes is.
 *            *total_nodes is the end of the last buffer.  When *total_nodes exceeds capacity_nodes nothing is written
 *            to nodes and every count is 0; *total_nodes still reports the nodes needed (the host form then returns
 *            RPL_RESULT_INSUFFICIENT_MEMORY).  Nothing at or past nodes + *total_nodes is written; the one padding
 *            node behind an odd-length buffer is unspecified.
 *   _dev:    device buffers, asynchronous on `stream` (NULL = the context's stream); nodes 16-byte aligned,
 *            node_offsets and total_nodes 8-byte, node_counts and status 4-byte aligned, else RPL_RESULT_INVALID_DATA.
 *            It waits for the session's last push (on any stream) and the session's next push waits for it; its scan
 *            kernels take turns with every other call of the context on its scan scratch.  No LaserScan is computed
 *            and nothing a push, a cloud or a message call returned is touched.
 *   host:    synchronous; copies back the tables, then only total_nodes * 8 bytes of nodes, chunked over the context's
 *            lanes as the host message calls are. */
rpl_result rpl_capsule_stream_nodes_dev(rpl_capsule_stream* s, uint32_t apply_ascend,
    const uint8_t* ascend_per_stream /* nullable, [n_streams], host */, rpl_node_hq* nodes, uint64_t capacity_nodes,
    uint64_t* node_offsets, uint32_t* node_counts, uint32_t* status, uint64_t* total_nodes, void* stream);
rpl_result rpl_capsule_stream_nodes(rpl_capsule_stream* s, uint32_t apply_ascend, const uint8_t* ascend_per_stream,
    rpl_node_hq* nodes, uint64_t capacity_nodes, uint64_t* node_offsets, uint32_t* node_counts, uint32_t* status,
    uint64_t* total_nodes);

/* Session messages: the serialised sensor_msgs/LaserScan and PointCloud2 (XCDR1, as rpl_*_cdr_batch_dev below) of
 * every scan the session's last successful push published, packed back to back, each ready for
 * rclcpp::SerializedMessage (INTEGRATION.md 4c) -- what scan_pub_->publish (src/rplidar_node.cpp:679) hands the RMW
 * layer, without the padded [n_streams * max_scans][max_nodes] arrays crossing the link.
 *   set_frames: per stream the message settings, synchronous: frame_ids [n_streams] (each at most 255 characters),
 *            range_max [n_streams] (nullable: keep the current values; the caller passes min(max_distance, hardware
 *            limit) per lidar, as rplidar_node.cpp:389-393).  Before the first call: "laser_frame" and 12.0f, the
 *            reference's defaults (rplidar_node.cpp:80, rplidar_node.hpp:328).
 *   Which scans, repeat calls, ordering and errors: those of the session clouds above.  Slot i = s * max_scans + k.
 *   laserscan_msgs[_dev]: slot k of stream s has a message iff k < min(scans_per_stream[s], max_scans) and its beam
 *            count is > 0 (the reference does not publish an empty scan, :609-611).  With B / E the slot's scan-begin
 *            stamp and the stamp of the scan-start node that closed it (the next scan's begin, whether that scan was
 *            published, dropped past max_scans or reset), SDK microseconds, 0 when unknown:
 *              ranges, intensities, angle_increment: what the push returned for the slot with the same params (the
 *                scan kernels run again on the scans where the session keeps them);
 *              header.stamp: t = B * 1000 + clock_offset_ns (int64 nanoseconds), sec = t / 10^9, nanosec = t % 10^9;
 *                {0, 0} when B == 0, t < 0 or sec > INT32_MAX;
 *              frame_id, range_max: the stream's settings; range_min 0.15f, angle_min 0.0f, angle_max (float)(2 pi);
 *              scan_duration = (double)((E - B) * 1000) / 1e9 (rclcpp Duration::seconds()), scan_time =
 *                (float)scan_duration, time_increment = (float)(scan_duration / denom), denom = beams in Mode A,
 *                max(beams - 1, 1) in Mode B (:635, :667); both 0 when B or E is 0 or E <= B.
 *            An unstamped push's messages have stamp {0, 0} and scan_time = time_increment = 0.
 *   cloud_msgs[_dev]: one message for every published slot (k < min(scans_per_stream[s], max_scans)), empty clouds
 *            included (the node publishes the cloud also when it drops the LaserScan): the session cloud of that slot
 *            (rpl_capsule_stream_cloud with the same params) as rpl_pointcloud2_cdr_batch_dev writes it, with the stamp and
 *            frame_id above.
 *   Packing: message i starts at msgs + msg_offsets[i], a multiple of 16 (msg_offsets [n_streams * max_scans] is the
 *            exclusive scan of the sizes, each rounded up to 16), msg_sizes[i] its bytes (0: no message), *total_bytes
 *            the end of the last message.  When *total_bytes exceeds capacity no message is written and every size is
 *            0; *total_bytes still reports the bytes needed (the host form then returns RPL_RESULT_INSUFFICIENT_MEMORY).
 *            Nothing at or past msgs + *total_bytes is written; the padding between messages is unspecified.
 *   _dev:    device buffers, asynchronous on `stream` (NULL = the context's stream); msgs 16-byte aligned, msg_offsets
 *            and total_bytes 8-byte, msg_sizes 4-byte aligned.  The session keeps a device block of its own for the
 *            scan outputs of every slot (8 bytes per node of max_nodes for LaserScan, 16 for PointCloud2), grown on
 *            the first call.
 *   host:    synchronous; copies back the tables, then only total_bytes of messages, chunked over the context's
 *            lanes as the host cloud call is. */
rpl_result rpl_capsule_stream_set_frames(rpl_capsule_stream* s, const char* const* frame_ids, const float* range_max);
rpl_result rpl_capsule_stream_laserscan_msgs_dev(rpl_capsule_stream* s, const rpl_scan_params* params,
                                                 int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                                 uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes,
                                                 void* stream);
rpl_result rpl_capsule_stream_laserscan_msgs(rpl_capsule_stream* s, const rpl_scan_params* params,
                                             int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                             uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes);
rpl_result rpl_capsule_stream_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_cloud_params* params,
                                             int64_t clock_offset_ns, uint8_t* msgs, uint64_t capacity,
                                             uint64_t* msg_offsets, uint32_t* msg_sizes, uint64_t* total_bytes,
                                             void* stream);
rpl_result rpl_capsule_stream_cloud_msgs(rpl_capsule_stream* s, const rpl_cloud_params* params, int64_t clock_offset_ns,
                                         uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                         uint64_t* total_bytes);

/* Messages from the push: one call that pushes `in` and returns the LaserScan messages of the scans it published,
 * written by the push's own scan kernels straight into the packed messages.  No padded
 * [n_streams * max_scans][max_nodes] row is allocated, computed into or copied.
 *   in:      one descriptor for every push flavour; the session's kind decides how data is read (framed: capsules
 *            [n_streams][stride_capsules][capsule bytes]; byte session: bytes [n_streams][stride_bytes]).  rx_us NULL:
 *            an unstamped push with sample_duration_us (rpl_capsule_stream_push / _push_bytes).  Else a stamped push
 *            with timing: capsule_rx_us (framed, rpl_capsule_stream_push_ts) or chunk_rx_us with chunk_bytes (byte
 *            session, rpl_capsule_stream_push_bytes_ts).  chunk_bytes must be 0 on a framed session and on an
 *            unstamped push.
 *   Definition: with two sessions of the same history, A pushed with the entry point of in's kind and then
 *            rpl_capsule_stream_laserscan_msgs[_dev] with params and clock_offset_ns, B with this call: for every slot
 *            i = s * max_scans + k, scans_per_stream and msg_sizes are equal, message i's msg_sizes[i] bytes are equal,
 *            and every later call returns on B what it returns on A (this call sets the last push as a push does).  A
 *            call that fails its checks leaves the session as the push it stands for would.
 *   Packing: the bound of slot i is rpl_laserscan_cdr_size(strlen(frame_id of s), n_i) rounded up to 16 for a
 *            published slot (k < min(scans_per_stream[s], max_scans); n_i its scan's node count, the node_counts[i]
 *            rpl_capsule_stream_nodes reports for the push), 0 for an unused one.  msg_offsets is the exclusive scan
 *            of the bounds in slot order and *total_bytes their sum: every message starts 16-byte aligned, and the
 *            bytes between a message's end and the next offset (8 per unmeasured node) are unspecified.  A message's
 *            exact size is only known once its scan kernel has run; its bound is known before, when each chunk's
 *            directory places its slots.
 *   Capacity: message i is written iff msg_offsets[i] + bound_i <= capacity, else its size is 0; the push itself is
 *            done either way.  Unlike laserscan_msgs this is not all or nothing: a device push's total is not known
 *            on the host before its chunks run.  The host form returns RPL_RESULT_INSUFFICIENT_MEMORY when
 *            *total_bytes > capacity, the _dev form reports it through *total_bytes only; in both cases
 *            rpl_capsule_stream_laserscan_msgs on the same push returns every message.  Nothing at or past
 *            msgs + min(*total_bytes, capacity) is written.
 *   Errors:  a null descriptor, data, counts, params, output or scans_per_stream; a stamped push with bad timing;
 *            misaligned device outputs; chunk_bytes where it does not belong; and the checks of the matching push
 *            and message calls: RPL_RESULT_INVALID_DATA.
 *   _dev:    data, counts, rx_us and the outputs are device memory (msgs 16-byte aligned, msg_offsets and total_bytes
 *            8-byte, msg_sizes and scans_per_stream 4-byte aligned); the descriptor and timing are host memory.
 *            Asynchronous on `stream` (NULL = the context's stream), ordered with the session's other calls as a
 *            device push is.
 *   host:    synchronous, host buffers.  Only the tables and the messages' stretch of msgs cross the link.
 *   Cost:    the session keeps, from the first call, 24 bytes per slot of device tables; the host form stages one
 *            chunk's bounded messages per lane instead of its padded rows. */
typedef struct rpl_push_input {
  const uint8_t* data;          /* framed session: capsules; byte session: bytes -- the session's kind decides */
  const uint32_t* counts;       /* [n_streams] capsules or bytes (the rules of the matching push) */
  const uint64_t* rx_us;        /* NULL: an unstamped push.  Else capsule_rx_us (framed) or chunk_rx_us (bytes), laid
                                   out as for push_ts / push_bytes_ts */
  const rpl_timing* timing;     /* stamped pushes (may be NULL with RPL_FLAG_PER_STREAM, as for push_ts) */
  uint32_t sample_duration_us;  /* unstamped pushes, as rpl_capsule_stream_push */
  uint32_t chunk_bytes;         /* stamped byte pushes, as rpl_capsule_stream_push_bytes_ts */
} rpl_push_input;
rpl_result rpl_capsule_stream_push_laserscan_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                                  const rpl_scan_params* params, int64_t clock_offset_ns, uint8_t* msgs,
                                                  uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                                  uint64_t* total_bytes, uint32_t* scans_per_stream);
rpl_result rpl_capsule_stream_push_laserscan_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                      const rpl_scan_params* params, int64_t clock_offset_ns,
                                                      uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                                      uint32_t* msg_sizes, uint64_t* total_bytes,
                                                      uint32_t* scans_per_stream, void* stream);

/* PointCloud2 messages from the push: one call that pushes `in` and returns the PointCloud2 messages of the scans it
 * published.  Each chunk of the push runs its cloud chain over the views its assembler has just made, then sizes and
 * packs the chunk's messages and writes them.  No LaserScan is computed, and no padded row of any kind crosses the link.
 *   in:      as rpl_capsule_stream_push_laserscan_msgs.
 *   params:  the cloud chain's, as rpl_capsule_stream_cloud_msgs.  With RPL_CLOUD_PER_STREAM the push decodes and stamps
 *            stream s with settings[s], as a push with RPL_FLAG_PER_STREAM does (of rpl_scan_params only that flag
 *            reaches the decoders, the assembler and the stamps), and its cloud takes settings[s].is_new_protocol.
 *            Without it the push takes in's timing for every stream.
 *   Definition: with two sessions of the same history, A pushed with the entry point of in's kind (RPL_FLAG_PER_STREAM
 *            iff params has RPL_CLOUD_PER_STREAM) and then rpl_capsule_stream_cloud_msgs[_dev] with params and
 *            clock_offset_ns, B with this call: when *total_bytes <= capacity, scans_per_stream, msg_offsets, msg_sizes,
 *            *total_bytes and every message's bytes are equal, and every later call returns on B what it returns on A
 *            (this call sets the last push as a push does).  A call that fails its checks leaves the session as the
 *            push it stands for would.
 *   Packing: exact, the packing of rpl_capsule_stream_cloud_msgs: slot i = s * max_scans + k of a published scan
 *            (k < min(scans_per_stream[s], max_scans)) has its message at the cloud's point count, an empty cloud
 *            included; an unused slot none.  msg_offsets is the exclusive scan of the sizes, each rounded up to 16, in
 *            slot order, and *total_bytes the end of the last message.  Unlike push_laserscan_msgs no bound is needed:
 *            each chunk sizes its messages after its cloud kernels have run, and a carry on the device continues the
 *            offsets from chunk to chunk.
 *   Capacity: message i is written iff msg_offsets[i] + its size <= capacity, else its size is 0: the written messages
 *            are a prefix, and the push itself is done either way.  Unlike cloud_msgs this is not all or nothing: a
 *            device push's total is not known on the host before its chunks run.  The host form returns
 *            RPL_RESULT_INSUFFICIENT_MEMORY when *total_bytes > capacity, the _dev form reports it through *total_bytes
 *            only; in both cases rpl_capsule_stream_cloud_msgs on the same push returns every message.  Nothing at or
 *            past msgs + min(*total_bytes, capacity) is written.
 *   Errors:  those of rpl_capsule_stream_push_laserscan_msgs, a params that fails the cloud chain's rules, and
 *            RPL_CLOUD_PER_STREAM before the first rpl_capsule_stream_set_lidars: RPL_RESULT_INVALID_DATA.
 *   _dev:    as rpl_capsule_stream_push_laserscan_msgs_dev.
 *   host:    synchronous, host buffers.  Only the tables and the messages' stretch of msgs cross the link.
 *   Cost:    the session keeps, from the first call, 24 bytes per slot of device tables.  The _dev form's clouds take a
 *            block of one device chunk's slots at max_nodes (16 bytes per node; the session's message work block, which
 *            cloud_msgs sizes for every slot); the host form stages one host chunk's clouds and messages per lane. */
rpl_result rpl_capsule_stream_push_cloud_msgs(rpl_capsule_stream* s, const rpl_push_input* in,
                                              const rpl_cloud_params* params, int64_t clock_offset_ns, uint8_t* msgs,
                                              uint64_t capacity, uint64_t* msg_offsets, uint32_t* msg_sizes,
                                              uint64_t* total_bytes, uint32_t* scans_per_stream);
rpl_result rpl_capsule_stream_push_cloud_msgs_dev(rpl_capsule_stream* s, const rpl_push_input* in,
                                                  const rpl_cloud_params* params, int64_t clock_offset_ns,
                                                  uint8_t* msgs, uint64_t capacity, uint64_t* msg_offsets,
                                                  uint32_t* msg_sizes, uint64_t* total_bytes,
                                                  uint32_t* scans_per_stream, void* stream);

/* Per-stream lidar settings: each stream of a session is one lidar, the reference's one RPlidarNode, with its own
 * intensity protocol (RealLidarDriver::is_new_type(), src/lidar_driver_wrapper.cpp:303-305), scan_processing and
 * inverted parameters (src/rplidar_node.cpp:270, 278-279) and SlamtecLidarTimingDesc (which depends on the model, the
 * scan mode and the link).  One session then serves a fleet that mixes them.
 *   set_lidars: synchronous (it waits for the session's device calls in flight that may read the table).  Copies
 *            settings[s] for every stream whose stream_mask entry is non-zero (NULL = all); the first call must set
 *            every stream.  A null settings, a first call that leaves a stream out, or a masked entry whose
 *            sample_duration_us is outside [1, 1000000] (the decoders' jump threshold divides by it):
 *            RPL_RESULT_INVALID_DATA, and the table is unchanged.
 *   RPL_FLAG_PER_STREAM in rpl_scan_params.flags (every push flavour: framed or byte, host or device, stamped or not;
 *            laserscan_msgs[_dev]): stream s is decoded, stamped and converted with settings[s] -- is_new_protocol,
 *            scan_processing, inverted, and timing for the decoder's discard threshold and the scan-begin stamps.  The
 *            call's own is_new_protocol, scan_processing, inverted, sample_duration_us and timing are ignored; timing
 *            may be NULL on a stamped push.  Each stream's outputs are bit for bit those of a session of that stream
 *            alone pushed with uniform params and timing equal to its settings.  Before the first set_lidars:
 *            RPL_RESULT_INVALID_DATA.
 *   RPL_CLOUD_PER_STREAM in rpl_cloud_params.flags (cloud[_dev], cloud_msgs[_dev]): stream s takes
 *            settings[s].is_new_protocol; before the first set_lidars: RPL_RESULT_INVALID_DATA.
 *   Changes between pushes apply to everything the next push decodes and publishes; a scan-begin stamp a push already
 *   computed (of a revolution still open) keeps its value.  Cloud and message calls read the table as it is when they
 *   are made.  apply_ascend stays a call parameter: it moves only unmeasured nodes, which the session nodes
 *   (rpl_capsule_stream_nodes*, below) alone keep, and they take it per call or per stream. */
typedef struct rpl_lidar_settings {
  uint8_t is_new_protocol; /* as rpl_scan_params */
  uint8_t scan_processing; /* 1 Mode A, 0 Mode B */
  uint8_t inverted;
  uint8_t pad;
  rpl_timing timing;       /* sample_duration_us must be in [1, 1000000] */
} rpl_lidar_settings;
rpl_result rpl_capsule_stream_set_lidars(rpl_capsule_stream* s, const rpl_lidar_settings* settings /* [n_streams] */,
                                         const uint8_t* stream_mask /* nullable: all */);

/* Per-stream clouds: each stream's PointCloud2 chain as its own node would run it (the NodeAccel parameters
 * publish_pointcloud, cloud_range_min / cloud_range_max, cloud_intensity_min, cloud_voxel_size, cloud_sor_k,
 * cloud_sor_alpha; INTEGRATION.md 4e), so that one session serves a fleet that mixes lidar models and cloud settings.
 *   set_clouds: synchronous (it waits for the session's device calls in flight).  Copies settings[s] for every stream
 *            whose stream_mask entry is non-zero (NULL = all); the first call must set every stream.  A null settings,
 *            a first call that leaves a stream out, or a masked entry that breaks the chain's rules (sor_k > 32; a
 *            voxel grid with voxel_size < 1e-6 or range_max >= 1000): RPL_RESULT_INVALID_DATA, and the table is
 *            unchanged.
 *   range_max 0: the stream's range_max of rpl_capsule_stream_set_frames, as it is when a cloud call is made (a
 *            set_frames in between moves the window).  A call whose resolved entry breaks the voxel rule:
 *            RPL_RESULT_INVALID_DATA.
 *   RPL_CLOUD_PER_STREAM_CHAIN in rpl_cloud_params.flags (cloud[_dev], cloud_msgs[_dev], push_cloud_msgs[_dev]): stream
 *            s takes range_min, range_max, intensity_min, voxel_size, sor_k and sor_alpha from its entry, and the call's
 *            own values of these six are ignored.  It combines with RPL_CLOUD_PER_STREAM (which still decides
 *            is_new_protocol) and RPL_CLOUD_NO_FUSED.  Before the first set_clouds: RPL_RESULT_INVALID_DATA.
 *   Definition: for an enabled stream every output of a flagged call -- point counts, xyzi rows, message sizes and
 *            bytes -- is bit for bit what a session of that stream alone gives on the same pieces with uniform
 *            rpl_cloud_params equal to its resolved entry.  A disabled stream (enabled 0) has point count 0 and its
 *            rows are not written (cloud[_dev]), and no message, size 0, as an unused slot (the message calls); its
 *            scans are not read.  A push still decodes, assembles and stamps it, so counters, carries and later calls
 *            are unchanged. */
typedef struct rpl_cloud_settings {
  float range_min;
  float range_max;      /* 0: the stream's range_max of rpl_capsule_stream_set_frames */
  float intensity_min;
  float voxel_size;     /* 0: no voxel grid */
  uint32_t sor_k;       /* 0: no statistical outlier removal; <= 32 */
  float sor_alpha;
  uint8_t enabled;      /* 0: this stream publishes no cloud */
  uint8_t pad[3];
} rpl_cloud_settings;   /* 28 bytes; the first 24 are laid out as in rpl_cloud_params */
rpl_result rpl_capsule_stream_set_clouds(rpl_capsule_stream* s, const rpl_cloud_settings* settings /* [n_streams] */,
                                         const uint8_t* stream_mask /* nullable: all */);

/* ---- LaserScan / PointCloud2 -> wire (SURVEY.md 8(f) rank 3) ---------------------------- */
/* The serialised message the RMW layer would produce from the message the reference publishes
 * (scan_pub_->publish, reference src/rplidar_node.cpp:679): XCDR1 little endian, 4-byte
 * encapsulation header, members in declaration order.  The host publishes the bytes as they are
 * (rclcpp::SerializedMessage, INTEGRATION.md 4c).  The reference tree holds no serialiser (it is in
 * the RMW dependency): the format follows the OMG CDR rules; parity unpinned. */
typedef struct rpl_laserscan_meta { /* sensor_msgs/LaserScan minus frame_id and the arrays */
  int32_t stamp_sec;
  uint32_t stamp_nanosec;
  float angle_min, angle_max, angle_increment, time_increment, scan_time, range_min, range_max;
} rpl_laserscan_meta;
uint32_t rpl_laserscan_cdr_size(uint32_t frame_id_len, uint32_t beam_count);
/* meta: [n_scans] on the device; angle_increment (nullable, device [n_scans]): the scan kernel's
 * output, overrides meta[s].angle_increment; ranges / intensities [n_scans][stride] and beam_counts
 * as rpl_scan_batch_dev wrote them.  cdr_out: [n_scans][cdr_stride] with cdr_stride % 4 == 0 and
 * cdr_stride >= rpl_laserscan_cdr_size(strlen(frame_id), stride); cdr_sizes (nullable): bytes used. */
rpl_result rpl_laserscan_cdr_batch_dev(rpl_ctx* ctx, const rpl_laserscan_meta* meta, const float* angle_increment,
                                       const char* frame_id, const float* ranges, const float* intensities,
                                       const uint32_t* beam_counts, uint32_t n_scans, uint32_t stride,
                                       uint8_t* cdr_out, uint32_t cdr_stride, uint32_t* cdr_sizes, void* stream);
uint32_t rpl_pointcloud2_cdr_size(uint32_t frame_id_len, uint32_t n_points);
/* sensor_msgs/PointCloud2 with fields x, y, z, intensity (float32, point_step 16, height 1, is_dense),
 * the layout laser_geometry produces and rpl_cloud_batch_dev writes.  stamps: device [n_clouds][2]
 * {sec, nanosec}; xyzi [n_clouds][stride][4]; cdr_stride % 16 == 0. */
rpl_result rpl_pointcloud2_cdr_batch_dev(rpl_ctx* ctx, const uint32_t* stamps, const char* frame_id,
                                         const float* xyzi, const uint32_t* point_counts, uint32_t n_clouds,
                                         uint32_t stride, uint8_t* cdr_out, uint32_t cdr_stride,
                                         uint32_t* cdr_sizes, void* stream);

/* ---- per-sample timestamps (SURVEY.md 8(f) rank 4) -------------------------------------- */
/* (rpl_timing is declared with the decoders above.) */
/* The stamp the SDK's unpackers attach to every node: receive time of a capsule minus
 * _getSampleDelayOffsetIn{Legacy,Express,HQ,UltraBoost,Dense,UltraDense}Mode (handler_normalnode.cpp:49-68,
 * handler_capsules.cpp:55-76,272-293,586-607,795-816, handler_hqnode.cpp:53-72).  capsule_rx_us:
 * [n_streams][stride_capsules] receive times; capsule_status / capsule_node_offset: the decoder's report;
 * node_ts_us: [n_streams][stride_capsules * rpl_capsule_nodes(ans_type)], written for released nodes. */
rpl_result rpl_node_timestamps_dev(rpl_ctx* ctx, uint32_t ans_type, const rpl_timing* timing,
                                   const uint64_t* capsule_rx_us, const uint32_t* capsule_status,
                                   const uint32_t* capsule_node_offset, const uint32_t* capsule_counts,
                                   uint32_t n_streams, uint32_t stride_capsules, uint64_t* node_ts_us, void* stream);
/* Standard nodes: the record ending at byte node_end[i] is stamped with the receive time of the
 * chunk_bytes-sized piece of the stream that byte arrived in (chunk_rx_us [n_streams][stride_chunks]). */
rpl_result rpl_normal_timestamps_dev(rpl_ctx* ctx, const rpl_timing* timing, const uint32_t* node_end,
                                     const uint32_t* node_counts, uint32_t n_streams, uint32_t stride_nodes,
                                     uint32_t chunk_bytes, const uint64_t* chunk_rx_us, uint32_t stride_chunks,
                                     uint64_t* node_ts_us, void* stream);

/* ---- synthetic scan streams (SURVEY.md 8(d)) ------------------------------------------ */
/* variant 0: tie-free rotated revolution, 5% unmeasured, quality 188; 1: same, quality
 * U[0,255]; 2: iid U[0,65535] keys (ties); 3: tie-free keys in pseudo-random order; 4: a
 * "room" (16 constant-range arcs of 2..10 m + 2 cm noise; non-trivial 5 cm voxels).
 * Also writes counts[s] = n when counts != NULL. */
rpl_result rpl_synth_batch_dev(rpl_ctx* ctx, uint64_t first_scan_id, uint32_t n_scans, uint32_t n,
                               uint32_t stride, int variant, rpl_node_hq* nodes, uint32_t* counts,
                               void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RPL_B200_H_ */
