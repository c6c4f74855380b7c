"""ctypes binding of librplidar_b200.so (include/rpl_b200.h) -- used by tests/ and bench.py.

This is a thin mirror of the C-ABI, not a second implementation: every call goes to the CUDA
library.  Loading fails loudly when the library has not been built (`build()` compiles it
in-tree with nvcc for sm_90a); creating a Context fails when no CUDA device is present.
There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# RPL_B200_LIB: alternative build of the same library (tuning experiments only)
LIB_PATH = os.environ.get("RPL_B200_LIB") or os.path.join(HERE, "librplidar_b200.so")

RESULT_OK = 0
RESULT_INVALID_DATA = 0x80008000
RESULT_OPERATION_FAIL = 0x80008001
RESULT_OPERATION_NOT_SUPPORT = 0x80008004
RESULT_INSUFFICIENT_MEMORY = 0x80008006
FLAG_FORCE_GENERAL = 1
FLAG_NO_TMA = 2
FLAG_NO_SMALL = 4
FLAG_PER_STREAM = 8
FLAG_PER_STREAM_FILTERS = 16
CLOUD_NO_FUSED = 1
CLOUD_PER_STREAM = 2
CLOUD_PER_STREAM_CHAIN = 4
CLOUD_PER_STREAM_FOOTPRINTS = 8
# rpl_scan_cloud_params.channels (laser_geometry ChannelOption)
SCAN_CLOUD_INTENSITY, SCAN_CLOUD_INDEX, SCAN_CLOUD_DISTANCE, SCAN_CLOUD_TIMESTAMP = 1, 2, 4, 8
# with a transform: the viewpoint channel, and the option that takes each stream's transform
SCAN_CLOUD_VIEWPOINT, SCAN_CLOUD_PER_STREAM_TRANSFORMS = 0x10, 0x100
CAPSULE_OK, CAPSULE_SYNC, CAPSULE_EMIT, CAPSULE_DISCARD = 1, 2, 4, 8
CAPSULE_CHECKSUM_ERR, CAPSULE_ENCODER_RESET_ERR, CAPSULE_BAD_FRAME = 16, 32, 64
PATH_FAST, PATH_GENERAL = 0, 1

# reference src/sdk/include/sl_lidar_cmd.h:272-278
NODE_DTYPE = np.dtype(
    {
        "names": ["angle_z_q14", "dist_mm_q2", "quality", "flag"],
        "formats": ["<u2", "<u4", "u1", "u1"],
        "offsets": [0, 2, 6, 7],
        "itemsize": 8,
    }
)

EXPORTS = [
    "rpl_abi_version", "rpl_ctx_create", "rpl_ctx_destroy", "rpl_last_error", "rpl_ctx_synchronize",
    "rpl_host_alloc", "rpl_host_free", "rpl_ctx_launch_count", "rpl_ctx_profile", "rpl_ctx_profile_read", "rpl_ascend_scan", "rpl_laserscan",
    "rpl_scan", "rpl_scan_batch", "rpl_ascend_scan_batch", "rpl_laserscan_batch", "rpl_scan_batch_dev",
    "rpl_cloud_batch_dev", "rpl_cloud_batch", "rpl_cloud_fuse_dev", "rpl_synth_batch_dev",
    "rpl_decode_dense_batch_dev", "rpl_decode_dense", "rpl_assemble_scans_dev", "rpl_assemble_scan_views_dev",
    "rpl_scan_views_dev", "rpl_chain_dense_laserscan", "rpl_decode_dense_batch_starts_dev",
    "rpl_assemble_scan_views_starts_dev",
    "rpl_capsule_stream_create", "rpl_capsule_stream_destroy", "rpl_capsule_stream_push", "rpl_capsule_stream_push_dev",
    "rpl_capsule_stream_reset", "rpl_capsule_stream_state", "rpl_capsule_stream_push_ts",
    "rpl_capsule_stream_push_ts_dev", "rpl_capsule_stream_counters",
    "rpl_capsule_stream_export", "rpl_capsule_stream_import",
    "rpl_capsule_stream_create_bytes", "rpl_capsule_stream_push_bytes", "rpl_capsule_stream_push_bytes_dev",
    "rpl_capsule_stream_create_bytes_mixed", "rpl_capsule_stream_set_answer_types",
    "rpl_capsule_stream_push_bytes_ts", "rpl_capsule_stream_push_bytes_ts_dev",
    "rpl_capsule_stream_cloud", "rpl_capsule_stream_cloud_dev", "rpl_capsule_stream_set_frames",
    "rpl_capsule_stream_set_lidars", "rpl_capsule_stream_set_clouds", "rpl_capsule_stream_laserscan_msgs", "rpl_capsule_stream_laserscan_msgs_dev",
    "rpl_capsule_stream_cloud_msgs", "rpl_capsule_stream_cloud_msgs_dev", "rpl_capsule_stream_nodes",
    "rpl_capsule_stream_nodes_dev", "rpl_capsule_stream_push_laserscan_msgs", "rpl_capsule_stream_push_laserscan_msgs_dev",
    "rpl_capsule_stream_push_cloud_msgs", "rpl_capsule_stream_push_cloud_msgs_dev",
    "rpl_scan_filter_batch_dev", "rpl_capsule_stream_set_scan_filters",
    "rpl_scan_filter_footprint_batch_dev", "rpl_capsule_stream_set_scan_footprints", "rpl_cloud_footprint_batch_dev",
    "rpl_scan_cloud_batch_dev", "rpl_capsule_stream_scan_cloud_msgs", "rpl_capsule_stream_scan_cloud_msgs_dev",
    "rpl_capsule_stream_push_scan_cloud_msgs", "rpl_capsule_stream_push_scan_cloud_msgs_dev",
    "rpl_capsule_stream_set_scan_cloud_transforms", "rpl_scan_cloud_transform_batch_dev",
    "rpl_rescan_batch_dev", "rpl_capsule_stream_set_rescans", "rpl_capsule_stream_rescan_msgs",
    "rpl_capsule_stream_rescan_msgs_dev",
    "rpl_rescan_window_batch_dev", "rpl_capsule_stream_set_rescan_windows", "rpl_capsule_stream_push_rescan_msgs",
    "rpl_capsule_stream_push_rescan_msgs_dev",
    "rpl_rescan_merge_batch_dev", "rpl_capsule_stream_set_rescan_merges", "rpl_capsule_stream_push_rescan_merge_msgs",
    "rpl_capsule_stream_push_rescan_merge_msgs_dev",
    "rpl_capsule_bytes", "rpl_capsule_nodes", "rpl_decode_capsules_batch_dev", "rpl_decode_capsules",
    "rpl_decode_normal_batch_dev", "rpl_decode_normal", "rpl_frame_capsules_dev", "rpl_node_timestamps_dev", "rpl_normal_timestamps_dev",
    "rpl_peer_gather_bytes", "rpl_peer_alloc", "rpl_peer_open", "rpl_peer_close", "rpl_peer_free",
    "rpl_cloud_fuse_push_dev",
    "rpl_exchange_unique_id", "rpl_exchange_create", "rpl_exchange_destroy", "rpl_exchange_allgather",
    "rpl_exchange_wait", "rpl_exchange_release", "rpl_exchange_slot", "rpl_exchange_synchronize",
    "rpl_laserscan_cdr_size", "rpl_laserscan_cdr_batch_dev", "rpl_pointcloud2_cdr_size", "rpl_pointcloud2_cdr_batch_dev",
]


class LaserScanMeta(C.Structure):
    """rpl_laserscan_meta: sensor_msgs/LaserScan minus frame_id and the arrays."""
    _fields_ = [("stamp_sec", C.c_int32), ("stamp_nanosec", C.c_uint32), ("angle_min", C.c_float),
                ("angle_max", C.c_float), ("angle_increment", C.c_float), ("time_increment", C.c_float),
                ("scan_time", C.c_float), ("range_min", C.c_float), ("range_max", C.c_float)]


LASERSCAN_META_DTYPE = np.dtype([("stamp_sec", "<i4"), ("stamp_nanosec", "<u4"), ("angle_min", "<f4"),
                                 ("angle_max", "<f4"), ("angle_increment", "<f4"), ("time_increment", "<f4"),
                                 ("scan_time", "<f4"), ("range_min", "<f4"), ("range_max", "<f4")])


class Timing(C.Structure):
    """rpl_timing == sl::SlamtecLidarTimingDesc without the bool."""
    _fields_ = [("sample_duration_us", C.c_uint32), ("native_baudrate", C.c_uint32),
                ("linkage_delay_us", C.c_uint32), ("native_interface_type", C.c_uint32)]


class LidarSettings(C.Structure):
    """rpl_lidar_settings: one stream's lidar (is_new_type(), scan_processing, inverted, timing)."""
    _fields_ = [("is_new_protocol", C.c_uint8), ("scan_processing", C.c_uint8), ("inverted", C.c_uint8),
                ("pad", C.c_uint8), ("timing", Timing)]


class ScanParams(C.Structure):
    _fields_ = [
        ("is_new_protocol", C.c_uint8),
        ("scan_processing", C.c_uint8),
        ("inverted", C.c_uint8),
        ("apply_ascend", C.c_uint8),
        ("flags", C.c_uint32),
    ]


class CloudParams(C.Structure):
    _fields_ = [
        ("range_min", C.c_float),
        ("range_max", C.c_float),
        ("intensity_min", C.c_float),
        ("voxel_size", C.c_float),
        ("sor_k", C.c_uint32),
        ("sor_alpha", C.c_float),
        ("is_new_protocol", C.c_uint8),
        ("flags", C.c_uint8),
        ("pad", C.c_uint8 * 2),
    ]


class CloudSettings(C.Structure):
    """rpl_cloud_settings: one stream's PointCloud2 chain (its node's publish_pointcloud and cloud_* parameters); the
    first 24 bytes are laid out as in CloudParams."""
    _fields_ = [
        ("range_min", C.c_float),
        ("range_max", C.c_float),
        ("intensity_min", C.c_float),
        ("voxel_size", C.c_float),
        ("sor_k", C.c_uint32),
        ("sor_alpha", C.c_float),
        ("enabled", C.c_uint8),
        ("pad", C.c_uint8 * 3),
    ]


class ScanFilterSettings(C.Structure):
    """rpl_scan_filter_settings: one LaserScan filter chain (angular mask, range window, intensity floor, speckle and
    veiling-point removal; 68 bytes).  oracle/scan_filter_oracle.py defines what it does."""
    _fields_ = [
        ("mask_lo", C.c_float * 4),
        ("mask_hi", C.c_float * 4),
        ("range_lo", C.c_float),
        ("range_hi", C.c_float),
        ("intensity_min", C.c_float),
        ("speckle_max_diff", C.c_float),
        ("shadow_angle", C.c_float),
        ("speckle_window", C.c_uint32),
        ("speckle_min_neighbours", C.c_uint32),
        ("shadow_window", C.c_uint32),
        ("enabled", C.c_uint8),
        ("pad", C.c_uint8 * 3),
    ]


class ScanFootprint(C.Structure):
    """rpl_scan_footprint: one stream's footprint, up to four polygons in the footprint frame with their invert bits and
    the pose of the LaserScan frame in that frame (544 bytes).  oracle/scan_footprint_oracle.py defines what it does."""
    _fields_ = [
        ("x", (C.c_float * 16) * 4),
        ("y", (C.c_float * 16) * 4),
        ("n_vertices", C.c_uint32 * 4),
        ("invert", C.c_uint8 * 4),
        ("pose_x", C.c_float),
        ("pose_y", C.c_float),
        ("pose_yaw", C.c_float),
    ]


class ScanCloudParams(C.Structure):
    """rpl_scan_cloud_params: the projection of LaserScans into PointCloud2 (laser_geometry's projectLaser; 8 bytes).
    oracle/scan_cloud_oracle.py defines what it does."""
    _fields_ = [("channels", C.c_uint32), ("range_cutoff", C.c_float)]


class ScanCloudTransform(C.Structure):
    """rpl_scan_cloud_transform: the pose of a published LaserScan frame in a target frame (geometry_msgs/Transform:
    translation, quaternion x, y, z, w) and whether it applies (64 bytes).  tests/scan_cloud_transform_oracle.py
    defines what it does."""
    _fields_ = [("translation", C.c_double * 3), ("rotation", C.c_double * 4), ("enabled", C.c_uint8),
                ("pad", C.c_uint8 * 7)]


class RescanSettings(C.Structure):
    """rpl_rescan_settings: one stream's re-gridded LaserScan, pointcloud_to_laserscan's parameters (40 bytes).
    oracle/rescan_oracle.py defines what it does."""
    _fields_ = [("angle_min", C.c_float), ("angle_max", C.c_float), ("angle_increment", C.c_float),
                ("range_min", C.c_float), ("range_max", C.c_float), ("min_height", C.c_float),
                ("max_height", C.c_float), ("inf_epsilon", C.c_float), ("scan_time", C.c_float),
                ("use_inf", C.c_uint8), ("enabled", C.c_uint8), ("pad", C.c_uint8 * 2)]


class RescanWindow(C.Structure):
    """rpl_rescan_window: one stream's window over its re-gridded LaserScans, laser_filters' LaserArrayFilter (8 bytes).
    oracle/rescan_window_oracle.py defines what it does."""
    _fields_ = [("observations", C.c_uint32), ("statistic", C.c_uint32)]


# rpl_stream_counters: one stream session stream's counters (include/rpl_b200.h)
STREAM_COUNTER_FIELDS = ("bytes_in", "frames", "skipped_bytes", "bad_frames", "checksum_errors", "encoder_resets",
                         "scan_resets", "discarded_capsules", "nodes", "nodes_unopened", "nodes_overwritten",
                         "scans_rewound", "scans_published", "scans_unreturned")
STREAM_COUNTERS_DTYPE = np.dtype([(f, "<u8") for f in STREAM_COUNTER_FIELDS])


class PushInput(C.Structure):
    """rpl_push_input: one push of any flavour for rpl_capsule_stream_push_{laserscan,cloud}_msgs[_dev] (addresses as
    ints)."""
    _fields_ = [("data", C.c_void_p), ("counts", C.c_void_p), ("rx_us", C.c_void_p), ("timing", C.POINTER(Timing)),
                ("sample_duration_us", C.c_uint32), ("chunk_bytes", C.c_uint32)]


class MsgsOut(C.Structure):
    """rpl_msgs_out: one packed message buffer and its tables (addresses as ints; 40 bytes)."""
    _fields_ = [("msgs", C.c_void_p), ("capacity", C.c_uint64), ("msg_offsets", C.c_void_p),
                ("msg_sizes", C.c_void_p), ("total_bytes", C.c_void_p)]


class RplError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rpl_result 0x{code:08x}: {msg}")
        self.code = code


def build(verbose: bool = False) -> str:
    """Compile librplidar_b200.so in-tree (nvcc, sm_90a)."""
    r = subprocess.run(["bash", os.path.join(HERE, "build.sh")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building librplidar_b200.so failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout)
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    """The loaded library.  Raises if it is not built: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: run rplidar_ros2_driver_b200/build.sh (or __graft_entry__.build()). "
            "The CUDA library is the only implementation of this path."
        )
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, sz, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_size_t, C.c_int
    PSP, PCP, PT = C.POINTER(ScanParams), C.POINTER(CloudParams), C.POINTER(Timing)
    sig = {
        "rpl_abi_version": ([], u32),
        "rpl_ctx_create": ([i32, u32, u32, C.POINTER(vp)], u32),
        "rpl_ctx_destroy": ([vp], None),
        "rpl_last_error": ([vp], C.c_char_p),
        "rpl_ctx_synchronize": ([vp], u32),
        "rpl_host_alloc": ([sz, C.POINTER(vp)], u32),
        "rpl_host_free": ([vp], None),
        "rpl_ctx_launch_count": ([vp], u64),
        "rpl_ctx_profile": ([vp, i32], u32),
        "rpl_ctx_profile_read": ([vp, C.POINTER(C.c_double), C.POINTER(u32), C.POINTER(C.c_double), C.POINTER(u32)], u32),
        "rpl_ascend_scan": ([vp, vp, sz], u32),
        "rpl_laserscan": ([vp, vp, sz, PSP, vp, vp, C.POINTER(u32), C.POINTER(C.c_float)], u32),
        "rpl_scan": ([vp, vp, sz, PSP, vp, vp, C.POINTER(u32), C.POINTER(C.c_float), C.POINTER(u32)], u32),
        "rpl_scan_batch": ([vp, vp, vp, u32, u32, PSP, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_ascend_scan_batch": ([vp, vp, vp, u32, u32, vp], u32),
        "rpl_laserscan_batch": ([vp, vp, vp, u32, u32, PSP, vp, vp, vp, vp], u32),
        "rpl_scan_batch_dev": ([vp, vp, vp, u32, u32, PSP, vp, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_cloud_batch_dev": ([vp, vp, vp, u32, u32, PCP, vp, vp, vp], u32),
        "rpl_cloud_footprint_batch_dev": ([vp, vp, vp, u32, u32, PCP, C.POINTER(ScanFootprint), vp, vp, vp], u32),
        "rpl_cloud_batch": ([vp, vp, vp, u32, u32, PCP, vp, vp], u32),
        "rpl_cloud_fuse_dev": ([vp, vp, vp, u32, u32, vp, vp, vp, vp], u32),
        "rpl_synth_batch_dev": ([vp, u64, u32, u32, u32, i32, vp, vp, vp], u32),
        "rpl_decode_dense_batch_dev": ([vp, vp, vp, u32, u32, u32, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_decode_dense": ([vp, vp, u32, u32, C.POINTER(u32), vp, C.POINTER(u32), vp, vp], u32),
        "rpl_capsule_bytes": ([u32], u32),
        "rpl_capsule_nodes": ([u32], u32),
        "rpl_decode_capsules_batch_dev": ([vp, u32, vp, vp, u32, u32, u32, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_decode_capsules": ([vp, u32, vp, u32, u32, vp, vp, C.POINTER(u32), vp, vp, vp, vp, vp], u32),
        "rpl_decode_normal_batch_dev": ([vp, vp, vp, u32, u32, vp, vp, vp, vp, vp], u32),
        "rpl_frame_capsules_dev": ([vp, u32, vp, vp, u32, u32, vp, u32, vp, vp, vp], u32),
        "rpl_peer_gather_bytes": ([u32, u32], C.c_size_t),
        "rpl_peer_alloc": ([vp, C.c_size_t, C.POINTER(vp), vp], u32),
        "rpl_peer_open": ([vp, vp, C.POINTER(vp)], u32),
        "rpl_peer_close": ([vp, vp], u32),
        "rpl_peer_free": ([vp, vp], u32),
        "rpl_cloud_fuse_push_dev": ([vp, vp, vp, u32, u32, vp, u32, u32, u32, vp, vp, vp], u32),
        "rpl_exchange_unique_id": ([vp], u32),
        "rpl_exchange_create": ([vp, vp, u32, u32, u32, u32, C.POINTER(vp)], u32),
        "rpl_exchange_destroy": ([vp], None),
        "rpl_exchange_allgather": ([vp, vp, vp, u32, u32, u32, vp, C.POINTER(u32)], u32),
        "rpl_exchange_wait": ([vp, u32, vp], u32),
        "rpl_exchange_release": ([vp, u32, vp], u32),
        "rpl_exchange_slot": ([vp, u32, u32, C.POINTER(vp), C.POINTER(vp)], u32),
        "rpl_exchange_synchronize": ([vp], u32),
        "rpl_laserscan_cdr_size": ([u32, u32], u32),
        "rpl_pointcloud2_cdr_size": ([u32, u32], u32),
        "rpl_laserscan_cdr_batch_dev": ([vp, vp, vp, C.c_char_p, vp, vp, vp, u32, u32, vp, u32, vp, vp], u32),
        "rpl_pointcloud2_cdr_batch_dev": ([vp, vp, C.c_char_p, vp, vp, u32, u32, vp, u32, vp, vp], u32),
        "rpl_node_timestamps_dev": ([vp, u32, C.POINTER(Timing), vp, vp, vp, vp, u32, u32, vp, vp], u32),
        "rpl_normal_timestamps_dev": ([vp, C.POINTER(Timing), vp, vp, u32, u32, u32, vp, u32, vp, vp], u32),
        "rpl_decode_normal": ([vp, vp, u32, vp, C.POINTER(u32)], u32),
        "rpl_assemble_scans_dev": ([vp, vp, vp, u32, u32, vp, vp, vp, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp], u32),
        "rpl_assemble_scan_views_dev": ([vp, vp, vp, u32, u32, vp, vp, vp, u32, u32, u32, vp, vp, vp, vp, vp, vp], u32),
        "rpl_scan_views_dev": ([vp, vp, u64, vp, u32, u32, PSP, vp, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_chain_dense_laserscan": ([vp, vp, vp, u32, u32, u32, PSP, u32, u32, vp, vp, vp, vp, vp], u32),
        "rpl_decode_dense_batch_starts_dev": ([vp, vp, vp, u32, u32, u32, vp, vp, vp, vp, vp, vp, vp, u32, vp, vp], u32),
        "rpl_assemble_scan_views_starts_dev": ([vp, vp, vp, u32, u32, vp, vp, vp, u32, vp, u32, vp, u32, u32, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_create": ([vp, u32, u32, u32, u32, u32, C.POINTER(vp)], u32),
        "rpl_capsule_stream_destroy": ([vp], None),
        "rpl_capsule_stream_push": ([vp, vp, vp, u32, PSP, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_dev": ([vp, vp, vp, u32, PSP, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_reset": ([vp, vp], u32),
        "rpl_capsule_stream_state": ([vp, vp, vp, vp], u32),
        "rpl_capsule_stream_counters": ([vp, vp, vp], u32),
        "rpl_capsule_stream_export": ([vp, vp, u32, vp, u64, vp, vp], u32),
        "rpl_capsule_stream_import": ([vp, vp, u32, vp, vp, u64], u32),
        "rpl_capsule_stream_push_ts": ([vp, vp, vp, PT, vp, PSP, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_ts_dev": ([vp, vp, vp, PT, vp, PSP, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_create_bytes": ([vp, u32, u32, u32, u32, u32, C.POINTER(vp)], u32),
        "rpl_capsule_stream_create_bytes_mixed": ([vp, vp, u32, u32, u32, u32, C.POINTER(vp)], u32),
        "rpl_capsule_stream_set_answer_types": ([vp, vp, vp], u32),
        "rpl_capsule_stream_push_bytes": ([vp, vp, vp, u32, PSP, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_bytes_dev": ([vp, vp, vp, u32, PSP, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_bytes_ts": ([vp, vp, vp, PT, u32, vp, PSP, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_bytes_ts_dev": ([vp, vp, vp, PT, u32, vp, PSP, vp, vp, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_cloud": ([vp, PCP, vp, vp], u32),
        "rpl_capsule_stream_cloud_dev": ([vp, PCP, vp, vp, vp], u32),
        "rpl_capsule_stream_set_frames": ([vp, vp, vp], u32),
        "rpl_capsule_stream_set_lidars": ([vp, vp, vp], u32),
        "rpl_capsule_stream_set_clouds": ([vp, vp, vp], u32),
        "rpl_capsule_stream_set_scan_filters": ([vp, vp, vp], u32),
        "rpl_scan_filter_batch_dev": ([vp, C.POINTER(ScanFilterSettings), vp, vp, vp, vp, u32, u32, vp], u32),
        "rpl_capsule_stream_set_scan_footprints": ([vp, vp, vp], u32),
        "rpl_scan_filter_footprint_batch_dev":
            ([vp, C.POINTER(ScanFilterSettings), C.POINTER(ScanFootprint), vp, vp, vp, vp, u32, u32, vp], u32),
        "rpl_scan_cloud_batch_dev": ([vp, C.POINTER(ScanCloudParams), vp, vp, vp, vp, vp, C.c_float, C.c_float, u32, u32,
                                      vp, vp, vp], u32),
        "rpl_scan_cloud_transform_batch_dev":
            ([vp, C.POINTER(ScanCloudParams), C.POINTER(ScanCloudTransform), vp, vp, vp, vp, vp, C.c_float, C.c_float,
              u32, u32, vp, vp, vp], u32),
        "rpl_capsule_stream_set_scan_cloud_transforms": ([vp, vp, vp, vp], u32),
        "rpl_rescan_batch_dev":
            ([vp, C.POINTER(RescanSettings), C.POINTER(ScanCloudParams), C.POINTER(ScanCloudTransform), vp, vp, vp, vp,
              C.c_float, C.c_float, u32, u32, vp, vp], u32),
        "rpl_capsule_stream_set_rescans": ([vp, vp, vp], u32),
        "rpl_capsule_stream_rescan_msgs":
            ([vp, PSP, C.POINTER(ScanCloudParams), C.c_int64, vp, u64, vp, vp, vp], u32),
        "rpl_capsule_stream_rescan_msgs_dev":
            ([vp, PSP, C.POINTER(ScanCloudParams), C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_scan_cloud_msgs":
            ([vp, PSP, C.POINTER(ScanCloudParams), C.c_int64, vp, u64, vp, vp, vp], u32),
        "rpl_capsule_stream_scan_cloud_msgs_dev":
            ([vp, PSP, C.POINTER(ScanCloudParams), C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_laserscan_msgs": ([vp, PSP, C.c_int64, vp, u64, vp, vp, vp], u32),
        "rpl_capsule_stream_laserscan_msgs_dev": ([vp, PSP, C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_cloud_msgs": ([vp, PCP, C.c_int64, vp, u64, vp, vp, vp], u32),
        "rpl_capsule_stream_cloud_msgs_dev": ([vp, PCP, C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_nodes": ([vp, u32, vp, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_nodes_dev": ([vp, u32, vp, vp, u64, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_laserscan_msgs": ([vp, C.POINTER(PushInput), PSP, C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_laserscan_msgs_dev":
            ([vp, C.POINTER(PushInput), PSP, C.c_int64, vp, u64, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_cloud_msgs": ([vp, C.POINTER(PushInput), PCP, C.c_int64, vp, u64, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_cloud_msgs_dev":
            ([vp, C.POINTER(PushInput), PCP, C.c_int64, vp, u64, vp, vp, vp, vp, vp], u32),
        "rpl_capsule_stream_push_scan_cloud_msgs":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), vp], u32),
        "rpl_capsule_stream_push_scan_cloud_msgs_dev":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), vp, vp], u32),
        "rpl_rescan_window_batch_dev": ([vp, C.POINTER(RescanWindow), vp, u32, u32, vp, vp], u32),
        "rpl_capsule_stream_set_rescan_windows": ([vp, vp, vp], u32),
        "rpl_capsule_stream_push_rescan_msgs":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), vp], u32),
        "rpl_capsule_stream_push_rescan_msgs_dev":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), vp, vp], u32),
        "rpl_rescan_merge_batch_dev": ([vp, C.POINTER(RescanSettings), vp, vp, u32, u32, vp, vp], u32),
        "rpl_capsule_stream_set_rescan_merges": ([vp, vp, vp, u32], u32),
        "rpl_capsule_stream_push_rescan_merge_msgs":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), C.POINTER(MsgsOut), vp], u32),
        "rpl_capsule_stream_push_rescan_merge_msgs_dev":
            ([vp, C.POINTER(PushInput), PSP, C.POINTER(ScanCloudParams), C.c_int64, C.POINTER(MsgsOut),
              C.POINTER(MsgsOut), C.POINTER(MsgsOut), vp, vp], u32),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name)  # AttributeError here = the library does not export the ABI
        fn.argtypes = args
        fn.restype = res
    _lib = L
    return L


def scan_params(is_new_protocol=0, scan_processing=1, inverted=0, apply_ascend=1, flags=0) -> ScanParams:
    return ScanParams(int(is_new_protocol), int(scan_processing), int(inverted), int(apply_ascend), int(flags))


def lidar_settings(is_new_protocol=0, scan_processing=1, inverted=0, timing: "Timing | None" = None) -> LidarSettings:
    """timing None: Timing(31, 0, 0, 0)"""
    return LidarSettings(int(is_new_protocol), int(scan_processing), int(inverted), 0,
                         timing if timing is not None else Timing(31, 0, 0, 0))


def cloud_params(range_min=0.15, range_max=40.0, intensity_min=0.0, voxel_size=0.0, sor_k=0,
                 sor_alpha=1.0, is_new_protocol=0, flags=0) -> CloudParams:
    return CloudParams(float(range_min), float(range_max), float(intensity_min), float(voxel_size),
                       int(sor_k), float(sor_alpha), int(is_new_protocol), int(flags), (C.c_uint8 * 2)(0, 0))


def cloud_settings(range_min=0.15, range_max=0.0, intensity_min=0.0, voxel_size=0.0, sor_k=0, sor_alpha=1.0,
                   enabled=True) -> CloudSettings:
    """range_max 0: the stream's range_max of set_frames."""
    return CloudSettings(float(range_min), float(range_max), float(intensity_min), float(voxel_size), int(sor_k),
                         float(sor_alpha), int(bool(enabled)), (C.c_uint8 * 3)(0, 0, 0))


def scan_filter_settings(mask=(), range_lo=float("-inf"), range_hi=float("inf"), intensity_min=float("-inf"),
                         speckle_window=0, speckle_min_neighbours=0, speckle_max_diff=0.0, shadow_window=0,
                         shadow_angle=0.0, enabled=True) -> ScanFilterSettings:
    """mask: up to four (lo, hi) sectors in radians (the others unused); the defaults remove nothing."""
    assert len(mask) <= 4
    lo = [float(a) for a, _ in mask] + [float("inf")] * (4 - len(mask))
    hi = [float(b) for _, b in mask] + [float("-inf")] * (4 - len(mask))
    return ScanFilterSettings((C.c_float * 4)(*lo), (C.c_float * 4)(*hi), float(range_lo), float(range_hi),
                              float(intensity_min), float(speckle_max_diff), float(shadow_angle), int(speckle_window),
                              int(speckle_min_neighbours), int(shadow_window), int(bool(enabled)),
                              (C.c_uint8 * 3)(0, 0, 0))


def scan_footprint(polygons=(), invert=(), pose=(0.0, 0.0, 0.0)) -> ScanFootprint:
    """polygons: up to four vertex lists [(x, y), ...] (3..16 vertices each, metres in the footprint frame); invert: a
    bit per polygon (missing: 0), set to remove what lies outside it; pose: (x, y, yaw) of the LaserScan frame in the
    footprint frame.  The defaults remove nothing."""
    assert len(polygons) <= 4 and len(invert) <= 4
    f = ScanFootprint()
    for p, poly in enumerate(polygons):
        f.n_vertices[p] = len(poly)
        for k, (x, y) in enumerate(poly):
            f.x[p][k], f.y[p][k] = float(x), float(y)
    for p, b in enumerate(invert):
        f.invert[p] = int(bool(b))
    f.pose_x, f.pose_y, f.pose_yaw = (float(v) for v in pose)
    return f


def scan_cloud_params(channels=SCAN_CLOUD_INTENSITY | SCAN_CLOUD_INDEX, range_cutoff=-1.0) -> ScanCloudParams:
    """laser_geometry's defaults: the intensity and index channels, range_cutoff -1 (each scan's range_max)."""
    return ScanCloudParams(int(channels), float(range_cutoff))


def scan_cloud_point_step(channels) -> int:
    """the bytes of one record: x, y, z, 4 per channel bit and 12 for the viewpoint"""
    return 12 + 4 * bin(int(channels) & 0xF).count("1") + (12 if int(channels) & SCAN_CLOUD_VIEWPOINT else 0)


def _scan_cloud_bound(channels, max_nodes) -> int:
    """the largest projected cloud message: the longest header (288), the tail (192; 264 with the viewpoint), the
    records of max_nodes beams and is_dense"""
    return 288 + (264 if int(channels) & SCAN_CLOUD_VIEWPOINT else 192) + scan_cloud_point_step(channels) * max_nodes + 1


def scan_cloud_transform(translation=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), enabled=True) -> ScanCloudTransform:
    """translation (x, y, z) in metres and the quaternion rotation (x, y, z, w) of the LaserScan frame in the target
    frame; enabled False: no transform (P as without one)."""
    return ScanCloudTransform((C.c_double * 3)(*(float(v) for v in translation)),
                              (C.c_double * 4)(*(float(v) for v in rotation)), int(bool(enabled)),
                              (C.c_uint8 * 7)())


FLT_MAX = float(np.finfo(np.float32).max)
RESCAN_MAX_BINS = 8192


def rescan_settings(angle_min=-math.pi, angle_max=math.pi, angle_increment=math.pi / 180.0, range_min=0.0,
                    range_max=FLT_MAX, min_height=-FLT_MAX, max_height=FLT_MAX, use_inf=True, inf_epsilon=1.0,
                    scan_time=1.0 / 30.0, enabled=True) -> RescanSettings:
    """pointcloud_to_laserscan's defaults for the angular grid, use_inf, inf_epsilon and scan_time; the range window
    and the height band default to everything a float holds (the package's double limits do not fit a float)."""
    return RescanSettings(float(angle_min), float(angle_max), float(angle_increment), float(range_min),
                          float(range_max), float(min_height), float(max_height), float(inf_epsilon),
                          float(scan_time), int(bool(use_inf)), int(bool(enabled)), (C.c_uint8 * 2)())


def rescan_ranges_size(settings: RescanSettings) -> int:
    """ranges_size of an entry: ceil(fl32(fl32(angle_max - angle_min) / angle_increment)) (0 outside [1, 8192])"""
    f = np.float32
    with np.errstate(all="ignore"):
        q = np.ceil(f(f(f(settings.angle_max) - f(settings.angle_min)) / f(settings.angle_increment)))
    return int(q) if 1 <= q <= RESCAN_MAX_BINS else 0


RESCAN_WINDOW_MEDIAN, RESCAN_WINDOW_MEAN = 0, 1
RESCAN_MERGE_NONE = 0xFFFFFFFF
RESCAN_WINDOW_MAX = 16


def rescan_window(observations=1, statistic="median") -> RescanWindow:
    """LaserArrayFilter's number_of_observations and its filter: "median" (MultiChannelMedianFilterFloat) or "mean"
    (MultiChannelMeanFilterFloat); observations 1 is no window."""
    stat = {"median": RESCAN_WINDOW_MEDIAN, "mean": RESCAN_WINDOW_MEAN}.get(statistic, statistic)
    return RescanWindow(int(observations), int(stat))


def _timing(t):
    return C.byref(t) if t is not None else None


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    return C.c_void_p(int(a))  # raw device / host address


class Context:
    """rpl_ctx wrapper.  One per thread (the reference has one scan thread per node)."""

    def __init__(self, device: int = 0, max_nodes: int = 8192, max_scans: int = 1):
        self._L = lib()
        h = C.c_void_p()
        rc = self._L.rpl_ctx_create(device, max_nodes, max_scans, C.byref(h))
        if rc != RESULT_OK:
            raise RplError(rc, "rpl_ctx_create failed (no CUDA device / not an H100?) -- there is no CPU fallback")
        self._h = h
        self.device, self.max_nodes, self.max_scans = device, max_nodes, max_scans

    def close(self):
        if getattr(self, "_h", None):
            self._L.rpl_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc: int):
        if rc != RESULT_OK:
            raise RplError(rc, (self._L.rpl_last_error(self._h) or b"").decode())

    def synchronize(self):
        self._check(self._L.rpl_ctx_synchronize(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._L.rpl_ctx_launch_count(self._h))

    def profile(self, enable: bool):
        self._check(self._L.rpl_ctx_profile(self._h, int(enable)))

    def profile_read(self):
        """(fast_ms, fast_launches, general_ms, general_launches) since the last read."""
        fm, gm, fn, gn = C.c_double(0), C.c_double(0), C.c_uint32(0), C.c_uint32(0)
        self._check(self._L.rpl_ctx_profile_read(self._h, C.byref(fm), C.byref(fn), C.byref(gm), C.byref(gn)))
        return fm.value, fn.value, gm.value, gn.value

    # ---- single scan (reference-shaped) ---------------------------------------------------
    def ascend_scan(self, nodes: np.ndarray):
        """ILidarDriver::ascendScanData: returns (sl_result, ascended copy)."""
        buf = np.ascontiguousarray(nodes, dtype=NODE_DTYPE).copy()
        rc = self._L.rpl_ascend_scan(self._h, _p(buf), buf.shape[0])
        return rc, buf

    def laserscan(self, nodes: np.ndarray, params: ScanParams):
        nodes = np.ascontiguousarray(nodes, dtype=NODE_DTYPE)
        n = nodes.shape[0]
        ranges = np.full(max(n, 1), np.nan, np.float32)
        inten = np.full(max(n, 1), np.nan, np.float32)
        beams, inc = C.c_uint32(0), C.c_float(0)
        self._check(self._L.rpl_laserscan(self._h, _p(nodes), n, C.byref(params), _p(ranges), _p(inten),
                                          C.byref(beams), C.byref(inc)))
        m = beams.value
        return ranges[:m].copy(), inten[:m].copy(), m, np.float32(inc.value)

    def scan(self, nodes: np.ndarray, params: ScanParams):
        """Fused grab glue + publish_scan.  Returns dict(nodes, ranges, intensities, beam_count,
        angle_increment, ascend_status)."""
        buf = np.ascontiguousarray(nodes, dtype=NODE_DTYPE).copy()
        n = buf.shape[0]
        ranges = np.full(max(n, 1), np.nan, np.float32)
        inten = np.full(max(n, 1), np.nan, np.float32)
        beams, inc, st = C.c_uint32(0), C.c_float(0), C.c_uint32(0)
        self._check(self._L.rpl_scan(self._h, _p(buf), n, C.byref(params), _p(ranges), _p(inten),
                                     C.byref(beams), C.byref(inc), C.byref(st)))
        m = beams.value
        return dict(nodes=buf, ranges=ranges[:m].copy(), intensities=inten[:m].copy(), beam_count=m,
                    angle_increment=np.float32(inc.value), ascend_status=st.value)

    # ---- batches, host buffers -----------------------------------------------------------------
    def scan_batch(self, nodes: np.ndarray, counts, params: ScanParams, emit_nodes=False, want_scan=True,
                   out=None):
        """nodes [n_scans, stride].  `out` may carry preallocated (e.g. pinned) arrays."""
        assert nodes.dtype == NODE_DTYPE and nodes.ndim == 2 and nodes.flags.c_contiguous
        n_scans, stride = nodes.shape
        counts = np.ascontiguousarray(counts, dtype=np.uint32)
        out = dict(out or {})
        # (no dict.setdefault here: it would build the default arrays even when they are given)
        if want_scan:
            for k in ("ranges", "intensities"):
                if k not in out:
                    out[k] = np.full((n_scans, stride), np.nan, np.float32)
        if emit_nodes and "nodes" not in out:
            out["nodes"] = np.zeros((n_scans, stride), NODE_DTYPE)
        for k, dt in (("beam_counts", np.uint32), ("angle_increment", np.float32), ("status", np.uint32),
                      ("path", np.uint32)):
            if k not in out:
                out[k] = np.zeros(n_scans, dt)
        self._check(self._L.rpl_scan_batch(
            self._h, _p(nodes), _p(counts), n_scans, stride, C.byref(params), _p(out.get("nodes")),
            _p(out.get("ranges")), _p(out.get("intensities")), _p(out["beam_counts"]),
            _p(out["angle_increment"]), _p(out["status"]), _p(out["path"])))
        return out

    # ---- batches, device buffers (addresses as ints, e.g. torch.Tensor.data_ptr()) -------------
    def scan_batch_dev(self, nodes, counts, n_scans, stride, params: ScanParams, nodes_out=None, ranges=None,
                       intensities=None, beam_counts=None, angle_increment=None, status=None, path=None,
                       stream=None):
        self._check(self._L.rpl_scan_batch_dev(
            self._h, _p(nodes), _p(counts), n_scans, stride, C.byref(params), _p(nodes_out), _p(ranges),
            _p(intensities), _p(beam_counts), _p(angle_increment), _p(status), _p(path), _p(stream)))

    def synth_batch_dev(self, first_scan_id, n_scans, n, stride, variant, nodes, counts=None, stream=None):
        self._check(self._L.rpl_synth_batch_dev(self._h, first_scan_id, n_scans, n, stride, variant, _p(nodes),
                                                _p(counts), _p(stream)))

    def cloud_batch_dev(self, nodes, counts, n_scans, stride, params: CloudParams, xyzi, point_counts, stream=None):
        self._check(self._L.rpl_cloud_batch_dev(self._h, _p(nodes), _p(counts), n_scans, stride, C.byref(params),
                                                _p(xyzi), _p(point_counts), _p(stream)))

    def cloud_footprint_batch_dev(self, nodes, counts, n_scans, stride, params: CloudParams,
                                  footprint: "ScanFootprint | None", xyzi, point_counts, stream=None):
        """cloud_batch_dev with one footprint (None: none) removing points before SOR and the voxel grid; its pose is
        the pose of the cloud's frame, nothing is mirrored."""
        self._check(self._L.rpl_cloud_footprint_batch_dev(
            self._h, _p(nodes), _p(counts), n_scans, stride, C.byref(params),
            C.byref(footprint) if footprint is not None else None, _p(xyzi), _p(point_counts), _p(stream)))

    def cloud_batch(self, nodes: np.ndarray, counts, params: CloudParams):
        assert nodes.dtype == NODE_DTYPE and nodes.ndim == 2 and nodes.flags.c_contiguous
        n_scans, stride = nodes.shape
        counts = np.ascontiguousarray(counts, dtype=np.uint32)
        xyzi = np.full((n_scans, stride, 4), np.nan, np.float32)
        pc = np.zeros(n_scans, np.uint32)
        self._check(self._L.rpl_cloud_batch(self._h, _p(nodes), _p(counts), n_scans, stride, C.byref(params),
                                            _p(xyzi), _p(pc)))
        return xyzi, pc

    # ---- dense-capsule decode (the step before the hot path) -------------------------------------
    def decode_dense(self, capsules: np.ndarray, sample_duration_us: int = 31, sync_state: int = 0):
        """One stream of framed capsules [n, 84] -> (nodes, capsule_status, capsule_node_offset, sync_state_out)."""
        capsules = np.ascontiguousarray(capsules, dtype=np.uint8).reshape(-1, 84)
        n = capsules.shape[0]
        nodes = np.zeros(max(40 * n, 1), NODE_DTYPE)
        status = np.zeros(max(n, 1), np.uint32)
        offs = np.zeros(max(n, 1), np.uint32)
        st, cnt = C.c_uint32(sync_state), C.c_uint32(0)
        self._check(self._L.rpl_decode_dense(self._h, _p(capsules), n, sample_duration_us, C.byref(st), _p(nodes),
                                             C.byref(cnt), _p(status), _p(offs)))
        return nodes[: cnt.value].copy(), status[:n].copy(), offs[:n].copy(), st.value

    def decode_dense_batch_dev(self, capsules, capsule_counts, n_streams, stride_capsules, sample_duration_us,
                               nodes_out, node_counts, sync_state_in=None, capsule_status=None,
                               capsule_node_offset=None, sync_state_out=None, stream=None, scan_starts=None,
                               starts_stride=0, scan_start_counts=None):
        if scan_starts is not None:
            self._check(self._L.rpl_decode_dense_batch_starts_dev(
                self._h, _p(capsules), _p(capsule_counts), n_streams, stride_capsules, sample_duration_us,
                _p(sync_state_in), _p(nodes_out), _p(node_counts), _p(capsule_status), _p(capsule_node_offset),
                _p(sync_state_out), _p(scan_starts), starts_stride, _p(scan_start_counts), _p(stream)))
            return
        self._check(self._L.rpl_decode_dense_batch_dev(
            self._h, _p(capsules), _p(capsule_counts), n_streams, stride_capsules, sample_duration_us,
            _p(sync_state_in), _p(nodes_out), _p(node_counts), _p(capsule_status), _p(capsule_node_offset),
            _p(sync_state_out), _p(stream)))

    # ---- the other answer formats (0x82 express, 0x83 HQ, 0x84 ultra, 0x86 ultra-dense, 0x81 standard) ----
    def decode_capsules(self, ans_type: int, capsules: np.ndarray, sample_duration_us: int = 31, state=(0, 0),
                        timing: "Timing | None" = None, capsule_rx_us=None):
        """One stream of framed capsules -> (nodes, capsule_status, capsule_node_offset, state_out); with
        timing + capsule_rx_us also the per-node timestamps as a fifth element."""
        cb, per = self._L.rpl_capsule_bytes(ans_type), self._L.rpl_capsule_nodes(ans_type)
        if cb == 0:
            raise ValueError(f"unknown answer type {ans_type:#x}")
        capsules = np.ascontiguousarray(capsules, dtype=np.uint8).reshape(-1, cb)
        n = capsules.shape[0]
        nodes = np.zeros(max(per * n, 1), NODE_DTYPE)
        status = np.zeros(max(n, 1), np.uint32)
        offs = np.zeros(max(n, 1), np.uint32)
        st = np.array(state, np.uint32)
        cnt = C.c_uint32(0)
        rx = ts = None
        if timing is not None:
            rx = np.ascontiguousarray(capsule_rx_us, dtype=np.uint64)
            ts = np.zeros(max(per * n, 1), np.uint64)
        self._check(self._L.rpl_decode_capsules(self._h, ans_type, _p(capsules), n, sample_duration_us, _p(st),
                                                _p(nodes), C.byref(cnt), _p(status), _p(offs),
                                                C.byref(timing) if timing is not None else None, _p(rx), _p(ts)))
        out = (nodes[: cnt.value].copy(), status[:n].copy(), offs[:n].copy(), (int(st[0]), int(st[1])))
        return out + (ts[: cnt.value].copy(),) if timing is not None else out

    def decode_capsules_batch_dev(self, ans_type, capsules, capsule_counts, n_streams, stride_capsules,
                                  sample_duration_us, nodes_out, node_counts, state_in=None, capsule_status=None,
                                  capsule_node_offset=None, state_out=None, stream=None):
        self._check(self._L.rpl_decode_capsules_batch_dev(
            self._h, ans_type, _p(capsules), _p(capsule_counts), n_streams, stride_capsules, sample_duration_us,
            _p(state_in), _p(nodes_out), _p(node_counts), _p(capsule_status), _p(capsule_node_offset),
            _p(state_out), _p(stream)))

    def frame_capsules_dev(self, ans_type, stream_bytes, byte_counts, n_streams, stride_bytes, capsules_out,
                           stride_capsules, capsule_counts_out, bytes_left_out=None, stream=None):
        self._check(self._L.rpl_frame_capsules_dev(
            self._h, ans_type, _p(stream_bytes), _p(byte_counts), n_streams, stride_bytes, _p(capsules_out),
            stride_capsules, _p(capsule_counts_out), _p(bytes_left_out), _p(stream)))

    def decode_normal(self, stream_bytes: np.ndarray):
        """Raw byte stream of 5-byte standard nodes -> nodes (byte-level resynchronisation included)."""
        b = np.ascontiguousarray(stream_bytes, dtype=np.uint8).reshape(-1)
        nodes = np.zeros(max(b.shape[0] // 5, 1), NODE_DTYPE)
        cnt = C.c_uint32(0)
        self._check(self._L.rpl_decode_normal(self._h, _p(b), b.shape[0], _p(nodes), C.byref(cnt)))
        return nodes[: cnt.value].copy()

    def decode_normal_batch_dev(self, stream_bytes, byte_counts, n_streams, stride_bytes, nodes_out, node_counts,
                                fsm_state_out=None, node_end=None, stream=None):
        self._check(self._L.rpl_decode_normal_batch_dev(
            self._h, _p(stream_bytes), _p(byte_counts), n_streams, stride_bytes, _p(nodes_out), _p(node_counts),
            _p(fsm_state_out), _p(node_end), _p(stream)))

    # ---- peer memory: fuse + all-gather in one kernel ---------------------------------------------------
    def peer_alloc(self, nbytes: int):
        """cudaMalloc + IPC handle: returns (device pointer, 64-byte handle)."""
        ptr = C.c_void_p()
        handle = np.zeros(64, np.uint8)
        self._check(self._L.rpl_peer_alloc(self._h, nbytes, C.byref(ptr), _p(handle)))
        return int(ptr.value), handle.tobytes()

    def peer_open(self, handle: bytes) -> int:
        h = np.frombuffer(handle, np.uint8).copy()
        ptr = C.c_void_p()
        self._check(self._L.rpl_peer_open(self._h, _p(h), C.byref(ptr)))
        return int(ptr.value)

    def peer_close(self, ptr: int):
        self._check(self._L.rpl_peer_close(self._h, C.c_void_p(ptr)))

    def peer_free(self, ptr: int):
        self._check(self._L.rpl_peer_free(self._h, C.c_void_p(ptr)))

    def cloud_fuse_push_dev(self, xyzi, point_counts, n_scans, stride, peer_bases, rank, slot_points, offsets, total,
                            stream=None):
        bases = (C.c_void_p * len(peer_bases))(*[C.c_void_p(int(b)) for b in peer_bases])
        self._check(self._L.rpl_cloud_fuse_push_dev(self._h, _p(xyzi), _p(point_counts), n_scans, stride, bases,
                                                    len(peer_bases), rank, slot_points, _p(offsets), _p(total),
                                                    _p(stream)))

    # ---- messages -> CDR (the step after the hot path) -----------------------------------------------
    def laserscan_cdr_batch_dev(self, meta, frame_id: str, ranges, intensities, beam_counts, n_scans, stride,
                                cdr_out, cdr_stride, cdr_sizes=None, angle_increment=None, stream=None):
        self._check(self._L.rpl_laserscan_cdr_batch_dev(
            self._h, _p(meta), _p(angle_increment), frame_id.encode(), _p(ranges), _p(intensities), _p(beam_counts),
            n_scans, stride, _p(cdr_out), cdr_stride, _p(cdr_sizes), _p(stream)))

    def pointcloud2_cdr_batch_dev(self, stamps, frame_id: str, xyzi, point_counts, n_clouds, stride, cdr_out,
                                  cdr_stride, cdr_sizes=None, stream=None):
        self._check(self._L.rpl_pointcloud2_cdr_batch_dev(
            self._h, _p(stamps), frame_id.encode(), _p(xyzi), _p(point_counts), n_clouds, stride, _p(cdr_out),
            cdr_stride, _p(cdr_sizes), _p(stream)))

    # ---- per-sample timestamps ---------------------------------------------------------------------
    def node_timestamps_dev(self, ans_type, timing: Timing, capsule_rx_us, capsule_status, capsule_node_offset,
                            capsule_counts, n_streams, stride_capsules, node_ts_us, stream=None):
        self._check(self._L.rpl_node_timestamps_dev(
            self._h, ans_type, C.byref(timing), _p(capsule_rx_us), _p(capsule_status), _p(capsule_node_offset),
            _p(capsule_counts), n_streams, stride_capsules, _p(node_ts_us), _p(stream)))

    def normal_timestamps_dev(self, timing: Timing, node_end, node_counts, n_streams, stride_nodes, chunk_bytes,
                              chunk_rx_us, stride_chunks, node_ts_us, stream=None):
        self._check(self._L.rpl_normal_timestamps_dev(
            self._h, C.byref(timing), _p(node_end), _p(node_counts), n_streams, stride_nodes, chunk_bytes,
            _p(chunk_rx_us), stride_chunks, _p(node_ts_us), _p(stream)))

    def assemble_scans_dev(self, nodes, node_counts, n_streams, stride_nodes, max_nodes, max_scans, scan_stride,
                           scans_out, scan_len, scans_per_stream, capsule_status=None, capsule_node_offset=None,
                           capsule_counts=None, stride_capsules=0, node_ts_us=None, scan_begin_ts_us=None,
                           stream=None):
        self._check(self._L.rpl_assemble_scans_dev(
            self._h, _p(nodes), _p(node_counts), n_streams, stride_nodes, _p(capsule_status), _p(capsule_node_offset),
            _p(capsule_counts), stride_capsules, max_nodes, max_scans, scan_stride, _p(scans_out), _p(scan_len),
            _p(scans_per_stream), _p(node_ts_us), _p(scan_begin_ts_us), _p(stream)))

    def assemble_scan_views_dev(self, nodes, node_counts, n_streams, stride_nodes, max_nodes, max_scans, views_out,
                                scan_len, scans_per_stream, capsule_status=None, capsule_node_offset=None,
                                capsule_counts=None, stride_capsules=0, node_ts_us=None, scan_begin_ts_us=None,
                                stream=None):
        self._check(self._L.rpl_assemble_scan_views_dev(
            self._h, _p(nodes), _p(node_counts), n_streams, stride_nodes, _p(capsule_status), _p(capsule_node_offset),
            _p(capsule_counts), stride_capsules, max_nodes, max_scans, _p(views_out), _p(scan_len),
            _p(scans_per_stream), _p(node_ts_us), _p(scan_begin_ts_us), _p(stream)))

    def assemble_scan_views_starts_dev(self, nodes, node_counts, n_streams, stride_nodes, scan_starts, starts_stride,
                                       scan_start_counts, max_nodes, max_scans, views_out, scan_len, scans_per_stream,
                                       capsule_status=None, capsule_node_offset=None, capsule_counts=None,
                                       stride_capsules=0, node_ts_us=None, scan_begin_ts_us=None, stream=None):
        self._check(self._L.rpl_assemble_scan_views_starts_dev(
            self._h, _p(nodes), _p(node_counts), n_streams, stride_nodes, _p(capsule_status), _p(capsule_node_offset),
            _p(capsule_counts), stride_capsules, _p(scan_starts), starts_stride, _p(scan_start_counts), max_nodes,
            max_scans, _p(views_out), _p(scan_len), _p(scans_per_stream), _p(node_ts_us), _p(scan_begin_ts_us),
            _p(stream)))

    def scan_views_dev(self, nodes, nodes_total, views, n_scans, stride, params: ScanParams, nodes_out=None, ranges=None,
                       intensities=None, beam_counts=None, angle_increment=None, status=None, path=None, stream=None):
        self._check(self._L.rpl_scan_views_dev(
            self._h, _p(nodes), nodes_total, _p(views), n_scans, stride, C.byref(params), _p(nodes_out), _p(ranges),
            _p(intensities), _p(beam_counts), _p(angle_increment), _p(status), _p(path), _p(stream)))

    def chain_dense_laserscan(self, capsules, capsule_counts, params: ScanParams, max_nodes, max_scans,
                              sample_duration_us=31, out=None):
        """Host buffers: capsules [n_streams, stride_capsules, 84] uint8 -> dict(ranges, intensities [n_streams*max_scans,
        max_nodes], beam_counts, angle_increment, scans_per_stream)."""
        assert capsules.dtype == np.uint8 and capsules.ndim == 3 and capsules.shape[2] == 84 and capsules.flags.c_contiguous
        n_streams, stride_caps = capsules.shape[:2]
        cc = np.ascontiguousarray(capsule_counts, dtype=np.uint32)
        out = dict(out or {})
        ns = n_streams * max_scans
        for k, shape, dt in (("ranges", (ns, max_nodes), np.float32), ("intensities", (ns, max_nodes), np.float32),
                             ("beam_counts", (ns,), np.uint32), ("angle_increment", (ns,), np.float32),
                             ("scans_per_stream", (n_streams,), np.uint32)):
            if k not in out:
                out[k] = np.zeros(shape, dt)
        self._check(self._L.rpl_chain_dense_laserscan(
            self._h, _p(capsules), _p(cc), n_streams, stride_caps, sample_duration_us, C.byref(params), max_nodes,
            max_scans, _p(out["ranges"]), _p(out["intensities"]), _p(out["beam_counts"]), _p(out["angle_increment"]),
            _p(out["scans_per_stream"])))
        return out

    def scan_filter_batch_dev(self, settings: ScanFilterSettings, ranges, intensities, beam_counts, angle_increment,
                              n_scans, stride, stream=None):
        """The LaserScan filters in place on rows of rpl_scan_batch_dev's layout (device addresses)."""
        self._check(self._L.rpl_scan_filter_batch_dev(self._h, C.byref(settings), _p(ranges), _p(intensities),
                                                      _p(beam_counts), _p(angle_increment), n_scans, stride,
                                                      _p(stream)))

    def scan_filter_footprint_batch_dev(self, settings: ScanFilterSettings, footprint: "ScanFootprint | None", ranges,
                                        intensities, beam_counts, angle_increment, n_scans, stride, stream=None):
        """scan_filter_batch_dev with a footprint (None: none)."""
        self._check(self._L.rpl_scan_filter_footprint_batch_dev(
            self._h, C.byref(settings), C.byref(footprint) if footprint is not None else None, _p(ranges),
            _p(intensities), _p(beam_counts), _p(angle_increment), n_scans, stride, _p(stream)))

    def scan_cloud_batch_dev(self, params: ScanCloudParams, ranges, intensities, beam_counts, angle_increment,
                             time_increment, range_min, range_max, n_scans, stride, points, point_counts, stream=None):
        """The projection of rows of rpl_scan_batch_dev's layout (device addresses; time_increment None: 0): scan s's
        point_step-byte records at points + s * stride * point_step, its kept count at point_counts[s]."""
        self._check(self._L.rpl_scan_cloud_batch_dev(
            self._h, C.byref(params), _p(ranges), _p(intensities), _p(beam_counts), _p(angle_increment),
            _p(time_increment), float(range_min), float(range_max), n_scans, stride, _p(points), _p(point_counts),
            _p(stream)))

    def scan_cloud_transform_batch_dev(self, params: ScanCloudParams, transform: "ScanCloudTransform | None", ranges,
                                       intensities, beam_counts, angle_increment, time_increment, range_min,
                                       range_max, n_scans, stride, points, point_counts, stream=None):
        """scan_cloud_batch_dev with every scan's points moved by one transform (None: none)."""
        self._check(self._L.rpl_scan_cloud_transform_batch_dev(
            self._h, C.byref(params), C.byref(transform) if transform is not None else None, _p(ranges),
            _p(intensities), _p(beam_counts), _p(angle_increment), _p(time_increment), float(range_min),
            float(range_max), n_scans, stride, _p(points), _p(point_counts), _p(stream)))

    def rescan_batch_dev(self, settings: RescanSettings, cloud_params: ScanCloudParams,
                         transform: "ScanCloudTransform | None", ranges, intensities, beam_counts, angle_increment,
                         range_min, range_max, n_scans, stride, out_ranges, stream=None):
        """The LaserScan re-gridded from the cloud scan_cloud_transform_batch_dev gives each row (device addresses;
        out_ranges [n_scans][rescan_ranges_size(settings)] float32; intensities may be None)."""
        self._check(self._L.rpl_rescan_batch_dev(
            self._h, C.byref(settings), C.byref(cloud_params), C.byref(transform) if transform is not None else None,
            _p(ranges), _p(intensities), _p(beam_counts), _p(angle_increment), float(range_min), float(range_max),
            n_scans, stride, _p(out_ranges), _p(stream)))

    def rescan_window_batch_dev(self, window: RescanWindow, in_ranges, n_scans, bins, out_ranges, stream=None):
        """Row t of out_ranges is the window's statistic over rows max(0, t - observations + 1) .. t of in_ranges
        (device addresses, [n_scans][bins] float32 each)."""
        self._check(self._L.rpl_rescan_window_batch_dev(self._h, C.byref(window), _p(in_ranges), n_scans, bins,
                                                        _p(out_ranges), _p(stream)))

    def rescan_merge_batch_dev(self, settings: RescanSettings, in_ranges, row_group, n_rows, n_groups, out_ranges,
                               stream=None):
        """Row g of out_ranges ([n_groups][ranges_size]) is the per-bin minimum, from the entry's seed, of the rows r of
        in_ranges ([n_rows][ranges_size]) with row_group[r] == g (device addresses; RESCAN_MERGE_NONE: no group)."""
        self._check(self._L.rpl_rescan_merge_batch_dev(self._h, C.byref(settings), _p(in_ranges), _p(row_group),
                                                       n_rows, n_groups, _p(out_ranges), _p(stream)))

    def cloud_fuse_dev(self, xyzi, point_counts, n_scans, stride, fused, offsets, total, stream=None):
        self._check(self._L.rpl_cloud_fuse_dev(self._h, _p(xyzi), _p(point_counts), n_scans, stride, _p(fused),
                                               _p(offsets), _p(total), _p(stream)))


class CapsuleStreamSession:
    """rpl_capsule_stream wrapper: capsules of one answer type (0x82 express, 0x83 HQ, 0x84 ultra, 0x85 dense, 0x86
    ultra-dense) pushed in pieces, scans published as the whole stream would publish them.  Borrows `ctx`; close it
    before the context."""

    def __init__(self, ctx: Context, ans_type: int, n_streams: int, stride_capsules: int, max_nodes: int, max_scans: int):
        self._init(ctx, ans_type, n_streams, stride_capsules, max_nodes, max_scans,
                   lambda h: ctx._L.rpl_capsule_stream_create(ctx._h, ans_type, n_streams, stride_capsules, max_nodes,
                                                               max_scans, C.byref(h)))

    def _init(self, ctx, ans_type, n_streams, stride_capsules, max_nodes, max_scans, create):
        self._L, self._ctx = ctx._L, ctx
        h = C.c_void_p()
        ctx._check(create(h))
        self._h = h
        self.ans_type, self.capsule_bytes = ans_type, int(self._L.rpl_capsule_bytes(ans_type))
        self.n_streams, self.stride_capsules, self.max_nodes, self.max_scans = n_streams, stride_capsules, max_nodes, max_scans

    def _fn(self, name):
        return getattr(self._L, f"rpl_capsule_stream_{name}")

    def close(self):
        if getattr(self, "_h", None):
            self._fn("destroy")(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _outputs(self, out):
        out = dict(out or {})
        ns = self.n_streams * self.max_scans
        for k, shape, dt in (("ranges", (ns, self.max_nodes), np.float32), ("intensities", (ns, self.max_nodes), np.float32),
                             ("beam_counts", (ns,), np.uint32), ("angle_increment", (ns,), np.float32),
                             ("scans_per_stream", (self.n_streams,), np.uint32)):
            if k not in out:
                out[k] = np.zeros(shape, dt)
        return out

    def _stamped_outputs(self, out):
        out = self._outputs(out)
        if "scan_begin_ts_us" not in out:
            out["scan_begin_ts_us"] = np.zeros(self.n_streams * self.max_scans, np.uint64)
        return out

    def push(self, capsules, capsule_counts, params: ScanParams, sample_duration_us=31, out=None, rx_us=None,
             timing: "Timing | None" = None):
        """Host buffers: capsules [n_streams, stride_capsules, capsule_bytes] uint8 -> the dict of
        Context.chain_dense_laserscan holding the scans this push published.  With rx_us ([n_streams, stride_capsules]
        receive time of every capsule) and timing, a stamped push (rpl_*_stream_push_ts, whose decoder takes
        timing.sample_duration_us): the dict also holds scan_begin_ts_us [n_streams * max_scans] uint64."""
        assert capsules.dtype == np.uint8 and capsules.shape == (self.n_streams, self.stride_capsules, self.capsule_bytes)
        assert capsules.flags.c_contiguous
        cc = np.ascontiguousarray(capsule_counts, dtype=np.uint32)
        assert cc.shape == (self.n_streams,)
        if rx_us is None and timing is None:
            out = self._outputs(out)
            self._ctx._check(self._fn("push")(
                self._h, _p(capsules), _p(cc), sample_duration_us, C.byref(params), _p(out["ranges"]),
                _p(out["intensities"]), _p(out["beam_counts"]), _p(out["angle_increment"]),
                _p(out["scans_per_stream"])))
            return out
        assert rx_us is not None and (timing is not None or params.flags & FLAG_PER_STREAM), \
            "a stamped push takes rx_us and timing (timing may be None with FLAG_PER_STREAM)"
        rx = np.ascontiguousarray(rx_us, dtype=np.uint64)
        assert rx.shape == (self.n_streams, self.stride_capsules)
        out = self._stamped_outputs(out)
        self._ctx._check(self._fn("push_ts")(
            self._h, _p(capsules), _p(cc), _timing(timing), _p(rx), C.byref(params), _p(out["ranges"]),
            _p(out["intensities"]), _p(out["beam_counts"]), _p(out["angle_increment"]), _p(out["scans_per_stream"]),
            _p(out["scan_begin_ts_us"])))
        return out

    def push_dev(self, capsules, capsule_counts, params: ScanParams, ranges, intensities, beam_counts,
                 angle_increment, scans_per_stream, sample_duration_us=31, stream=None, rx_us=None,
                 timing: "Timing | None" = None, scan_begin_ts_us=None):
        """Device addresses (the layouts of push), asynchronous on `stream` (None: the context's stream).  With rx_us,
        timing and scan_begin_ts_us (device addresses but timing), a stamped push."""
        if rx_us is None and timing is None and scan_begin_ts_us is None:
            self._ctx._check(self._fn("push_dev")(
                self._h, _p(capsules), _p(capsule_counts), sample_duration_us, C.byref(params), _p(ranges),
                _p(intensities), _p(beam_counts), _p(angle_increment), _p(scans_per_stream), _p(stream)))
            return
        self._ctx._check(self._fn("push_ts_dev")(
            self._h, _p(capsules), _p(capsule_counts), C.byref(timing) if timing is not None else None, _p(rx_us),
            C.byref(params), _p(ranges), _p(intensities), _p(beam_counts), _p(angle_increment), _p(scans_per_stream),
            _p(scan_begin_ts_us), _p(stream)))

    def cloud(self, params: CloudParams, out=None):
        """The PointCloud2 chain over the scans the last push published, read where the session keeps them:
        {"xyzi": [n_streams * max_scans, max_nodes, 4] float32, "point_counts": [n_streams * max_scans] uint32}, slot k
        of stream s the cloud of the scan in slot k of that push's outputs (unused slots: count 0, row untouched)."""
        out = dict(out or {})
        ns = self.n_streams * self.max_scans
        if "xyzi" not in out:
            out["xyzi"] = np.zeros((ns, self.max_nodes, 4), np.float32)
        if "point_counts" not in out:
            out["point_counts"] = np.zeros(ns, np.uint32)
        assert out["xyzi"].shape == (ns, self.max_nodes, 4) and out["xyzi"].dtype == np.float32
        assert out["point_counts"].shape == (ns,) and out["point_counts"].dtype == np.uint32
        self._ctx._check(self._fn("cloud")(self._h, C.byref(params), _p(out["xyzi"]), _p(out["point_counts"])))
        return out

    def cloud_dev(self, params: CloudParams, xyzi, point_counts, stream=None):
        """Device addresses (the layouts of cloud), asynchronous on `stream` (None: the context's stream)."""
        self._ctx._check(self._fn("cloud_dev")(self._h, C.byref(params), _p(xyzi), _p(point_counts), _p(stream)))

    def set_frames(self, frame_ids, range_max=None):
        """Per stream the frame_id and LaserScan range_max of the messages (range_max None: keep the current ones)."""
        assert len(frame_ids) == self.n_streams
        ids = (C.c_char_p * self.n_streams)(*[f.encode() for f in frame_ids])
        rm = None if range_max is None else np.ascontiguousarray(range_max, dtype=np.float32)
        assert rm is None or rm.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_frames")(self._h, C.cast(ids, C.c_void_p), _p(rm)))

    def set_lidars(self, settings, mask=None):
        """Per stream the lidar's settings (n_streams LidarSettings, see lidar_settings) that pushes and message calls
        with FLAG_PER_STREAM, and cloud calls with CLOUD_PER_STREAM, use.  Only the entries where mask is true are
        copied (None: all); the first call must set every stream."""
        assert len(settings) == self.n_streams
        arr = (LidarSettings * self.n_streams)(*settings)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_lidars")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_clouds(self, settings, mask=None):
        """Per stream the PointCloud2 chain (n_streams CloudSettings, see cloud_settings) that cloud calls with
        CLOUD_PER_STREAM_CHAIN use instead of their params' window, SOR and voxel grid.  Only the entries where mask is
        true are copied (None: all); the first call must set every stream."""
        assert len(settings) == self.n_streams
        arr = (CloudSettings * self.n_streams)(*settings)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_clouds")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_scan_filters(self, settings, mask=None):
        """Per stream the LaserScan filters (n_streams ScanFilterSettings, see scan_filter_settings) that pushes and
        LaserScan message calls with FLAG_PER_STREAM_FILTERS apply.  Only the entries where mask is true are copied
        (None: all); the first call must set every stream."""
        assert len(settings) == self.n_streams
        arr = (ScanFilterSettings * self.n_streams)(*settings)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_scan_filters")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_scan_footprints(self, footprints, mask=None):
        """Per stream the footprint (n_streams ScanFootprint, see scan_footprint) that the filters of calls with
        FLAG_PER_STREAM_FILTERS apply as one of their stages, and cloud calls with CLOUD_PER_STREAM_FOOTPRINTS before
        SOR and the voxel grid (an inverted stream's cloud, with CLOUD_PER_STREAM, against the mirrored polygons).
        Only the entries where mask is true are copied (None: all); the first call must set every stream."""
        assert len(footprints) == self.n_streams
        arr = (ScanFootprint * self.n_streams)(*footprints)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_scan_footprints")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_scan_cloud_transforms(self, transforms, target_frames, mask=None):
        """Per stream the transform (n_streams ScanCloudTransform, see scan_cloud_transform) and target frame (str; None
        for a disabled entry) of the clouds that projecting calls with SCAN_CLOUD_PER_STREAM_TRANSFORMS publish.  Only
        the entries where mask is true are copied (None: all); the first call must set every stream."""
        assert len(transforms) == self.n_streams and len(target_frames) == self.n_streams
        arr = (ScanCloudTransform * self.n_streams)(*transforms)
        names = (C.c_char_p * self.n_streams)(*(None if f is None else f.encode() for f in target_frames))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_scan_cloud_transforms")(self._h, C.cast(arr, C.c_void_p),
                                                                C.cast(names, C.c_void_p), _p(m)))

    def set_rescans(self, settings, mask=None):
        """Per stream the re-gridded LaserScan (n_streams RescanSettings, see rescan_settings) that rescan_msgs[_dev]
        publish.  Only the entries where mask is true are copied (None: all); the first call must set every stream."""
        assert len(settings) == self.n_streams
        arr = (RescanSettings * self.n_streams)(*settings)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_rescans")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_rescan_windows(self, windows, mask=None):
        """Per stream the window over the re-gridded LaserScans push_rescan_msgs[_dev] publish (n_streams RescanWindow,
        see rescan_window).  Only the entries where mask is true are copied (None: all), and their windows start
        over; until the first call every stream has observations 1."""
        assert len(windows) == self.n_streams
        arr = (RescanWindow * self.n_streams)(*windows)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_rescan_windows")(self._h, C.cast(arr, C.c_void_p), _p(m)))

    def set_rescan_merges(self, group_of_stream, max_age):
        """The groups whose re-gridded scans push_rescan_merge_msgs[_dev] merge into one LaserScan each: per stream its
        group (< len(max_age)) or RESCAN_MERGE_NONE, and per group how many merge pushes a member's grid is kept for.
        Replaces every group; every held grid starts empty."""
        g = np.ascontiguousarray(group_of_stream, dtype=np.uint32)
        assert g.shape == (self.n_streams,)
        a = np.ascontiguousarray(max_age, dtype=np.uint32).reshape(-1)
        self._ctx._check(self._fn("set_rescan_merges")(self._h, _p(g), _p(a) if a.size else None, int(a.size)))

    def _msgs(self, name, params, clock_offset_ns, msgs, packed, cloud_params=None):
        ns = self.n_streams * self.max_scans
        if msgs is None:  # room for every slot's largest message
            if name == "laserscan_msgs":
                per = 288 + 32 + 8 * self.max_nodes + 4
            elif name == "scan_cloud_msgs":
                per = _scan_cloud_bound(cloud_params.channels, self.max_nodes)
            elif name == "rescan_msgs":
                per = 288 + 36 + 4 * RESCAN_MAX_BINS
            else:
                per = 288 + 116 + 16 * self.max_nodes + 1
            msgs = np.zeros(ns * ((per + 15) // 16 * 16), np.uint8)
        assert msgs.dtype == np.uint8 and msgs.flags.c_contiguous
        offs, sizes, total = np.zeros(ns, np.uint64), np.zeros(ns, np.uint32), np.zeros(1, np.uint64)
        extra = () if cloud_params is None else (C.byref(cloud_params),)
        rc = self._fn(name)(self._h, C.byref(params), *extra, int(clock_offset_ns), _p(msgs), msgs.size, _p(offs),
                            _p(sizes), _p(total))
        if not packed or rc != RESULT_INSUFFICIENT_MEMORY:
            self._ctx._check(rc)
        if packed:
            return dict(msgs=msgs, msg_offsets=offs, msg_sizes=sizes, total_bytes=int(total[0]), result=rc)
        return [bytes(msgs[o: o + s]) if s else None for o, s in zip(offs.tolist(), sizes.tolist())]

    def laserscan_msgs(self, params: ScanParams, clock_offset_ns=0, msgs=None, packed=False):
        """The serialised sensor_msgs/LaserScan of every scan the last push published: per slot (n_streams *
        max_scans) the message's bytes, None for no message.  msgs: the host buffer to pack into (its size is the
        capacity; None: one that always fits).  packed: return {"msgs", "msg_offsets", "msg_sizes", "total_bytes",
        "result"} instead, with result RESULT_INSUFFICIENT_MEMORY rather than an exception when msgs is too small."""
        return self._msgs("laserscan_msgs", params, clock_offset_ns, msgs, packed)

    def cloud_msgs(self, params: CloudParams, clock_offset_ns=0, msgs=None, packed=False):
        """The serialised sensor_msgs/PointCloud2 of every published slot, as laserscan_msgs."""
        return self._msgs("cloud_msgs", params, clock_offset_ns, msgs, packed)

    def scan_cloud_msgs(self, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns=0, msgs=None,
                        packed=False):
        """The serialised sensor_msgs/PointCloud2 projected from every LaserScan message laserscan_msgs(params) gives
        (laser_geometry's projectLaser with cloud_params), as laserscan_msgs returns them."""
        return self._msgs("scan_cloud_msgs", params, clock_offset_ns, msgs, packed, cloud_params)

    def scan_cloud_msgs_dev(self, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns, msgs, capacity,
                            msg_offsets, msg_sizes, total_bytes, stream=None):
        """Device addresses, as laserscan_msgs_dev."""
        self._ctx._check(self._fn("scan_cloud_msgs_dev")(
            self._h, C.byref(params), C.byref(cloud_params), int(clock_offset_ns), _p(msgs), int(capacity),
            _p(msg_offsets), _p(msg_sizes), _p(total_bytes), _p(stream)))

    def rescan_msgs(self, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns=0, msgs=None,
                    packed=False):
        """The serialised sensor_msgs/LaserScan re-gridded (pointcloud_to_laserscan, with each stream's set_rescans
        entry) from every cloud scan_cloud_msgs(params, cloud_params) gives, as laserscan_msgs returns them."""
        return self._msgs("rescan_msgs", params, clock_offset_ns, msgs, packed, cloud_params)

    def rescan_msgs_dev(self, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns, msgs, capacity,
                        msg_offsets, msg_sizes, total_bytes, stream=None):
        """Device addresses, as laserscan_msgs_dev."""
        self._ctx._check(self._fn("rescan_msgs_dev")(
            self._h, C.byref(params), C.byref(cloud_params), int(clock_offset_ns), _p(msgs), int(capacity),
            _p(msg_offsets), _p(msg_sizes), _p(total_bytes), _p(stream)))

    def laserscan_msgs_dev(self, params: ScanParams, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                           total_bytes, stream=None):
        """Device addresses (msgs [capacity] bytes, msg_offsets [n_streams * max_scans] uint64, msg_sizes uint32,
        total_bytes one uint64), asynchronous on `stream` (None: the context's stream)."""
        self._ctx._check(self._fn("laserscan_msgs_dev")(self._h, C.byref(params), int(clock_offset_ns), _p(msgs),
                                                         int(capacity), _p(msg_offsets), _p(msg_sizes),
                                                         _p(total_bytes), _p(stream)))

    def cloud_msgs_dev(self, params: CloudParams, clock_offset_ns, msgs, capacity, msg_offsets, msg_sizes,
                       total_bytes, stream=None):
        """Device addresses, as laserscan_msgs_dev."""
        self._ctx._check(self._fn("cloud_msgs_dev")(self._h, C.byref(params), int(clock_offset_ns), _p(msgs),
                                                     int(capacity), _p(msg_offsets), _p(msg_sizes), _p(total_bytes),
                                                     _p(stream)))

    def _push_input(self, data, counts, sample_duration_us, rx_us, timing, chunk_bytes):
        t = None if timing is None else C.pointer(timing)
        pi = PushInput(_p(data).value if data is not None else None, _p(counts).value if counts is not None else None,
                       _p(rx_us).value if rx_us is not None else None, t, sample_duration_us, chunk_bytes or 0)
        pi._keep = t
        return pi

    def _push_msgs(self, name, data, counts, params, clock_offset_ns, sample_duration_us, rx_us, timing, chunk_bytes,
                   msgs, packed):
        assert isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.flags.c_contiguous
        cnt = np.ascontiguousarray(counts, dtype=np.uint32)
        assert cnt.shape == (self.n_streams,)
        rx = None if rx_us is None else np.ascontiguousarray(rx_us, dtype=np.uint64)
        ns = self.n_streams * self.max_scans
        if msgs is None:  # room for every slot's largest message
            per = 288 + (32 + 8 * self.max_nodes + 4 if name == "push_laserscan_msgs" else 116 + 16 * self.max_nodes + 1)
            msgs = np.zeros(ns * ((per + 15) // 16 * 16), np.uint8)
        assert msgs.dtype == np.uint8 and msgs.flags.c_contiguous
        offs, sizes, total = np.zeros(ns, np.uint64), np.zeros(ns, np.uint32), np.zeros(1, np.uint64)
        sps = np.zeros(self.n_streams, np.uint32)
        pi = self._push_input(data, cnt, sample_duration_us, rx, timing, chunk_bytes)
        rc = self._fn(name)(self._h, C.byref(pi), C.byref(params), int(clock_offset_ns), _p(msgs), msgs.size, _p(offs),
                            _p(sizes), _p(total), _p(sps))
        if not packed or rc != RESULT_INSUFFICIENT_MEMORY:
            self._ctx._check(rc)
        if packed:
            return dict(msgs=msgs, msg_offsets=offs, msg_sizes=sizes, total_bytes=int(total[0]), result=rc), sps
        return [bytes(msgs[o: o + n]) if n else None for o, n in zip(offs.tolist(), sizes.tolist())], sps

    def push_laserscan_msgs(self, data, counts, params: ScanParams, clock_offset_ns=0, sample_duration_us=31,
                            rx_us=None, timing: "Timing | None" = None, chunk_bytes=None, msgs=None, packed=False):
        """One push (host buffers: data and counts as the push of the session's kind; rx_us -- capsule receive times on a
        framed session, chunk receive times with chunk_bytes on a byte session -- and timing: a stamped push) whose
        scans come back as their serialised sensor_msgs/LaserScan, written by the push's scan kernels.  Returns
        (messages, scans_per_stream): messages as laserscan_msgs returns them (per slot the bytes or None; packed: the
        dict, with the push's own bound-based offsets and result RESULT_INSUFFICIENT_MEMORY rather than an exception
        when msgs is too small -- the push is done either way).  msgs None: a buffer that always fits."""
        return self._push_msgs("push_laserscan_msgs", data, counts, params, clock_offset_ns, sample_duration_us, rx_us,
                               timing, chunk_bytes, msgs, packed)

    def push_laserscan_msgs_dev(self, data, counts, params: ScanParams, clock_offset_ns, msgs, capacity, msg_offsets,
                                msg_sizes, total_bytes, scans_per_stream, sample_duration_us=31, rx_us=None,
                                timing: "Timing | None" = None, chunk_bytes=None, stream=None):
        """Device addresses (data, counts, rx_us and the outputs, laid out as for push_laserscan_msgs and
        laserscan_msgs_dev), asynchronous on `stream` (None: the context's stream)."""
        pi = self._push_input(data, counts, sample_duration_us, rx_us, timing, chunk_bytes)
        self._ctx._check(self._fn("push_laserscan_msgs_dev")(
            self._h, C.byref(pi), C.byref(params), int(clock_offset_ns), _p(msgs), int(capacity), _p(msg_offsets),
            _p(msg_sizes), _p(total_bytes), _p(scans_per_stream), _p(stream)))

    def push_cloud_msgs(self, data, counts, params: CloudParams, clock_offset_ns=0, sample_duration_us=31, rx_us=None,
                        timing: "Timing | None" = None, chunk_bytes=None, msgs=None, packed=False):
        """One push, as push_laserscan_msgs takes it, whose scans come back as their serialised sensor_msgs/PointCloud2:
        each chunk of the push runs the cloud chain of params over its scans, then packs their messages exactly as
        cloud_msgs does.  With CLOUD_PER_STREAM the push decodes and stamps each stream with its own lidar settings.
        Returns (messages, scans_per_stream) as push_laserscan_msgs; capacity is per message (the written messages
        are a prefix), and RESULT_INSUFFICIENT_MEMORY (packed) leaves the push done."""
        return self._push_msgs("push_cloud_msgs", data, counts, params, clock_offset_ns, sample_duration_us, rx_us,
                               timing, chunk_bytes, msgs, packed)

    def push_cloud_msgs_dev(self, data, counts, params: CloudParams, clock_offset_ns, msgs, capacity, msg_offsets,
                            msg_sizes, total_bytes, scans_per_stream, sample_duration_us=31, rx_us=None,
                            timing: "Timing | None" = None, chunk_bytes=None, stream=None):
        """Device addresses, as push_laserscan_msgs_dev."""
        pi = self._push_input(data, counts, sample_duration_us, rx_us, timing, chunk_bytes)
        self._ctx._check(self._fn("push_cloud_msgs_dev")(
            self._h, C.byref(pi), C.byref(params), int(clock_offset_ns), _p(msgs), int(capacity), _p(msg_offsets),
            _p(msg_sizes), _p(total_bytes), _p(scans_per_stream), _p(stream)))

    def _push_msgs_sets(self, name, second_bytes, data, counts, params, cloud_params, clock_offset_ns,
                        sample_duration_us, rx_us, timing, chunk_bytes, msgs, second_msgs, merged=None, n_groups=None):
        """A push returning packed message sets (entry point `name`): the LaserScans into msgs, the second set into
        second_msgs; None: a buffer that always fits, second_bytes per slot for the second set.  With n_groups (a merge
        push) a third set, by group, into merged (None: one that always fits)."""
        assert isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.flags.c_contiguous
        cnt = np.ascontiguousarray(counts, dtype=np.uint32)
        assert cnt.shape == (self.n_streams,)
        rx = None if rx_us is None else np.ascontiguousarray(rx_us, dtype=np.uint64)
        ns = self.n_streams * self.max_scans
        if msgs is None:
            msgs = np.zeros(ns * ((288 + 32 + 8 * self.max_nodes + 4 + 15) // 16 * 16), np.uint8)
        if second_msgs is None:
            second_msgs = np.zeros(ns * ((second_bytes + 15) // 16 * 16), np.uint8)
        bufs = [(msgs, ns), (second_msgs, ns)]
        if n_groups is not None:
            if merged is None:
                merged = np.zeros(max(n_groups, 1) * ((second_bytes + 15) // 16 * 16), np.uint8)
            bufs.append((merged, n_groups))
        out = []
        for buf, n in bufs:
            assert buf.dtype == np.uint8 and buf.flags.c_contiguous
            t = dict(msgs=buf, msg_offsets=np.zeros(n, np.uint64), msg_sizes=np.zeros(n, np.uint32),
                     total=np.zeros(1, np.uint64))
            t["out"] = MsgsOut(_p(buf).value, buf.size, _p(t["msg_offsets"]).value, _p(t["msg_sizes"]).value,
                               _p(t["total"]).value)
            out.append(t)
        sps = np.zeros(self.n_streams, np.uint32)
        pi = self._push_input(data, cnt, sample_duration_us, rx, timing, chunk_bytes)
        rc = self._fn(name)(self._h, C.byref(pi), C.byref(params), C.byref(cloud_params), int(clock_offset_ns),
                            *[C.byref(t["out"]) for t in out], _p(sps))
        if rc != RESULT_INSUFFICIENT_MEMORY:
            self._ctx._check(rc)
        res = [dict(msgs=t["msgs"], msg_offsets=t["msg_offsets"], msg_sizes=t["msg_sizes"],
                    total_bytes=int(t["total"][0]), result=rc) for t in out]
        return (*res, sps)

    def push_scan_cloud_msgs(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns=0,
                             sample_duration_us=31, rx_us=None, timing: "Timing | None" = None, chunk_bytes=None,
                             msgs=None, cloud_msgs=None):
        """One push, as push_laserscan_msgs takes it, whose scans come back both as their serialised
        sensor_msgs/LaserScan and as the PointCloud2 each projects to (laser_geometry's projectLaser with
        cloud_params), from one run of the scan kernels.  msgs / cloud_msgs: the host buffers to pack into (their sizes
        are the capacities; None: ones that always fit).  Returns (scans, clouds, scans_per_stream): scans and clouds
        as the packed dicts of push_laserscan_msgs(packed=True), each with the call's result, which is
        RESULT_INSUFFICIENT_MEMORY rather than an exception when either buffer is too small (the push is done)."""
        return self._push_msgs_sets("push_scan_cloud_msgs", _scan_cloud_bound(cloud_params.channels, self.max_nodes),
                                    data, counts, params, cloud_params, clock_offset_ns, sample_duration_us, rx_us,
                                    timing, chunk_bytes, msgs, cloud_msgs)

    def push_scan_cloud_msgs_dev(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams,
                                 clock_offset_ns, scans: MsgsOut, clouds: MsgsOut, scans_per_stream,
                                 sample_duration_us=31, rx_us=None, timing: "Timing | None" = None, chunk_bytes=None,
                                 stream=None):
        """Device addresses (data, counts, rx_us and scans_per_stream as for push_laserscan_msgs_dev; scans and clouds
        MsgsOut of device buffers laid out as for laserscan_msgs_dev), asynchronous on `stream` (None: the context's
        stream)."""
        pi = self._push_input(data, counts, sample_duration_us, rx_us, timing, chunk_bytes)
        self._ctx._check(self._fn("push_scan_cloud_msgs_dev")(
            self._h, C.byref(pi), C.byref(params), C.byref(cloud_params), int(clock_offset_ns), C.byref(scans),
            C.byref(clouds), _p(scans_per_stream), _p(stream)))

    def push_rescan_msgs(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns=0,
                         sample_duration_us=31, rx_us=None, timing: "Timing | None" = None, chunk_bytes=None,
                         msgs=None, rescan_msgs=None):
        """One push, as push_laserscan_msgs takes it, whose scans come back both as their serialised
        sensor_msgs/LaserScan and as the LaserScan each re-grids to (rescan_msgs with cloud_params), windowed per
        stream by set_rescan_windows.  Buffers and returns (scans, rescans, scans_per_stream) as
        push_scan_cloud_msgs."""
        return self._push_msgs_sets("push_rescan_msgs", 288 + 36 + 4 * RESCAN_MAX_BINS, data, counts, params,
                                    cloud_params, clock_offset_ns, sample_duration_us, rx_us, timing, chunk_bytes, msgs,
                                    rescan_msgs)

    def push_rescan_msgs_dev(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams, clock_offset_ns,
                             scans: MsgsOut, rescans: MsgsOut, scans_per_stream, sample_duration_us=31, rx_us=None,
                             timing: "Timing | None" = None, chunk_bytes=None, stream=None):
        """Device addresses, as push_scan_cloud_msgs_dev."""
        pi = self._push_input(data, counts, sample_duration_us, rx_us, timing, chunk_bytes)
        self._ctx._check(self._fn("push_rescan_msgs_dev")(
            self._h, C.byref(pi), C.byref(params), C.byref(cloud_params), int(clock_offset_ns), C.byref(scans),
            C.byref(rescans), _p(scans_per_stream), _p(stream)))

    def push_rescan_merge_msgs(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams, n_groups,
                               clock_offset_ns=0, sample_duration_us=31, rx_us=None, timing: "Timing | None" = None,
                               chunk_bytes=None, msgs=None, rescan_msgs=None, merged_msgs=None):
        """push_rescan_msgs, plus one merged LaserScan per group of set_rescan_merges (n_groups of them) that has news:
        the per-bin minimum of the members' held grids.  Returns (scans, rescans, merged, scans_per_stream), merged
        packed by group as the others by slot."""
        return self._push_msgs_sets("push_rescan_merge_msgs", 288 + 36 + 4 * RESCAN_MAX_BINS, data, counts, params,
                                    cloud_params, clock_offset_ns, sample_duration_us, rx_us, timing, chunk_bytes, msgs,
                                    rescan_msgs, merged_msgs, n_groups)

    def push_rescan_merge_msgs_dev(self, data, counts, params: ScanParams, cloud_params: ScanCloudParams,
                                   clock_offset_ns, scans: MsgsOut, rescans: MsgsOut, merged: MsgsOut,
                                   scans_per_stream, sample_duration_us=31, rx_us=None,
                                   timing: "Timing | None" = None, chunk_bytes=None, stream=None):
        """Device addresses, as push_rescan_msgs_dev; merged is indexed by group."""
        pi = self._push_input(data, counts, sample_duration_us, rx_us, timing, chunk_bytes)
        self._ctx._check(self._fn("push_rescan_merge_msgs_dev")(
            self._h, C.byref(pi), C.byref(params), C.byref(cloud_params), int(clock_offset_ns), C.byref(scans),
            C.byref(rescans), C.byref(merged), _p(scans_per_stream), _p(stream)))

    def nodes(self, apply_ascend=True, per_stream=None, packed=False, nodes=None):
        """The node buffers RealLidarDriver::grab_scan_data would return for every scan the last push published: per
        slot (n_streams * max_scans) an array of NODE_DTYPE (empty for an unused slot), ascended when apply_ascend, or,
        with per_stream ([n_streams] flags), where the stream's flag is set.  nodes: the host buffer to pack into
        (None: one that always fits).  packed: return {"nodes", "node_offsets", "node_counts", "status",
        "total_nodes", "result"} instead, with result RESULT_INSUFFICIENT_MEMORY rather than an exception when nodes is
        too small; otherwise (buffers, status)."""
        ns = self.n_streams * self.max_scans
        if nodes is None:
            nodes = np.zeros(ns * self.max_nodes, NODE_DTYPE)
        assert nodes.dtype == NODE_DTYPE and nodes.flags.c_contiguous
        m = None if per_stream is None else np.ascontiguousarray(per_stream, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        offs, counts, status = np.zeros(ns, np.uint64), np.zeros(ns, np.uint32), np.zeros(ns, np.uint32)
        total = np.zeros(1, np.uint64)
        rc = self._fn("nodes")(self._h, int(bool(apply_ascend)), _p(m), _p(nodes), nodes.size, _p(offs), _p(counts),
                               _p(status), _p(total))
        if not packed or rc != RESULT_INSUFFICIENT_MEMORY:
            self._ctx._check(rc)
        if packed:
            return dict(nodes=nodes, node_offsets=offs, node_counts=counts, status=status, total_nodes=int(total[0]),
                        result=rc)
        return [nodes[o: o + n] for o, n in zip(offs.tolist(), counts.tolist())], status

    def nodes_dev(self, nodes, capacity_nodes, node_offsets, node_counts, status, total_nodes, apply_ascend=True,
                  per_stream=None, stream=None):
        """Device addresses (nodes [capacity_nodes] 8-byte nodes, node_offsets [n_streams * max_scans] uint64,
        node_counts and status uint32, total_nodes one uint64; per_stream a host array), asynchronous on `stream`
        (None: the context's stream)."""
        m = None if per_stream is None else np.ascontiguousarray(per_stream, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("nodes_dev")(self._h, int(bool(apply_ascend)), _p(m), _p(nodes), int(capacity_nodes),
                                               _p(node_offsets), _p(node_counts), _p(status), _p(total_nodes),
                                               _p(stream)))

    def reset(self, mask=None):
        """Drops the held capsule, the decoder state and the open revolution of the streams where mask is true
        (None: every stream)."""
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("reset")(self._h, _p(m)))

    def state(self):
        """(open_nodes, held_capsule): nodes in each stream's open revolution, 1 where a valid capsule is held."""
        open_nodes = np.zeros(self.n_streams, np.uint32)
        held = np.zeros(self.n_streams, np.uint32)
        self._ctx._check(self._fn("state")(self._h, _p(open_nodes), _p(held), None))
        return open_nodes, held

    def counters(self, clear=None):
        """Every stream's counters since create (or since its last clear), after every push issued before the call:
        a STREAM_COUNTERS_DTYPE array [n_streams].  clear ([n_streams] flags, None: none): the streams whose counters
        are zeroed after the copy."""
        out = np.zeros(self.n_streams, STREAM_COUNTERS_DTYPE)
        m = None if clear is None else np.ascontiguousarray(clear, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("counters")(self._h, _p(out), _p(m)))
        return out

    def export_streams(self, streams):
        """The carried state and counters of the listed streams as records (rpl_capsule_stream_export): (records
        uint8 [total_bytes], offsets uint64 [len(streams)]), record i at records[offsets[i]:].  The session is left as
        it was; import_streams puts the records into any session of the same kind and max_nodes."""
        s = np.ascontiguousarray(streams, dtype=np.uint32).reshape(-1)
        offsets, total = np.zeros(s.size, np.uint64), np.zeros(1, np.uint64)
        rc = self._fn("export")(self._h, _p(s), s.size, None, 0, _p(offsets), _p(total))
        if rc != RESULT_INSUFFICIENT_MEMORY or s.size == 0:
            self._ctx._check(rc)
        records = np.zeros(int(total[0]), np.uint8)
        self._ctx._check(self._fn("export")(self._h, _p(s), s.size, _p(records), records.size, _p(offsets), _p(total)))
        return records, offsets

    def import_streams(self, streams, records, offsets):
        """Stream streams[i] takes record i of export_streams' (records, offsets) (rpl_capsule_stream_import); its
        settings, the other streams and the last push's outputs are left alone.  A record that does not fit the
        session raises RplError (RESULT_INVALID_DATA) and changes nothing."""
        s = np.ascontiguousarray(streams, dtype=np.uint32).reshape(-1)
        r = np.ascontiguousarray(records, dtype=np.uint8).reshape(-1)
        o = np.ascontiguousarray(offsets, dtype=np.uint64).reshape(-1)
        assert o.size == s.size
        self._ctx._check(self._fn("import")(self._h, _p(s), s.size, _p(r) if r.size else None, _p(o), r.size))
        if hasattr(self, "ans_types"):  # a mixed session's streams take their records' types
            for i, off in zip(s.tolist(), o.tolist()):
                self.ans_types[i] = int(r[off + 12: off + 16].view(np.uint32)[0])


class DenseStreamSession(CapsuleStreamSession):
    """The capsule session fixed to dense capsules (0x85, 84 bytes)."""

    def __init__(self, ctx: Context, n_streams: int, stride_capsules: int, max_nodes: int, max_scans: int):
        super().__init__(ctx, 0x85, n_streams, stride_capsules, max_nodes, max_scans)


class CapsuleByteStreamSession(CapsuleStreamSession):
    """rpl_capsule_stream byte session (rpl_capsule_stream_create_bytes): the raw serial bytes of a measurement answer
    type (0x81..0x86, after the answer descriptor) pushed in any pieces, with the unpackers' search for the sync bytes
    (0x81: the unfinished record) carried across pushes; scans published as the whole stream would publish them.  close
    and reset are the capsule session's; state() returns (open_nodes, held_capsule, held_bytes), held_bytes = bytes of
    the unfinished frame (0x81: record) held for the next push."""

    def __init__(self, ctx: Context, ans_type: int, n_streams: int, stride_bytes: int, max_nodes: int, max_scans: int):
        self._init(ctx, ans_type, n_streams, 0, max_nodes, max_scans,
                   lambda h: ctx._L.rpl_capsule_stream_create_bytes(ctx._h, ans_type, n_streams, stride_bytes, max_nodes,
                                                                     max_scans, C.byref(h)))
        self.stride_bytes = stride_bytes

    def push(self, stream_bytes, byte_counts, params: ScanParams, sample_duration_us=31, out=None, chunk_bytes=None,
             chunk_rx_us=None, timing: "Timing | None" = None):
        """Host buffers: stream_bytes [n_streams, stride_bytes] uint8 -> the dict of CapsuleStreamSession.push.  With
        chunk_bytes, chunk_rx_us ([n_streams, ceil(stride_bytes / chunk_bytes)]: receive time of each chunk_bytes piece
        of this push) and timing, a stamped push (whose decoder takes timing.sample_duration_us): the dict also holds
        scan_begin_ts_us."""
        assert stream_bytes.dtype == np.uint8 and stream_bytes.shape == (self.n_streams, self.stride_bytes)
        assert stream_bytes.flags.c_contiguous
        bc = np.ascontiguousarray(byte_counts, dtype=np.uint32)
        assert bc.shape == (self.n_streams,)
        if chunk_bytes is None and chunk_rx_us is None and timing is None:
            out = self._outputs(out)
            self._ctx._check(self._L.rpl_capsule_stream_push_bytes(
                self._h, _p(stream_bytes), _p(bc), sample_duration_us, C.byref(params), _p(out["ranges"]),
                _p(out["intensities"]), _p(out["beam_counts"]), _p(out["angle_increment"]),
                _p(out["scans_per_stream"])))
            return out
        assert chunk_bytes is not None and chunk_rx_us is not None and (timing is not None or params.flags & FLAG_PER_STREAM), \
            "a stamped push takes chunk_bytes, chunk_rx_us and timing (timing may be None with FLAG_PER_STREAM)"
        rx = np.ascontiguousarray(chunk_rx_us, dtype=np.uint64)
        assert chunk_bytes == 0 or rx.shape == (self.n_streams, -(-self.stride_bytes // chunk_bytes))
        out = self._stamped_outputs(out)
        self._ctx._check(self._L.rpl_capsule_stream_push_bytes_ts(
            self._h, _p(stream_bytes), _p(bc), _timing(timing), chunk_bytes, _p(rx), C.byref(params),
            _p(out["ranges"]), _p(out["intensities"]), _p(out["beam_counts"]), _p(out["angle_increment"]),
            _p(out["scans_per_stream"]), _p(out["scan_begin_ts_us"])))
        return out

    def push_dev(self, stream_bytes, byte_counts, params: ScanParams, ranges, intensities, beam_counts,
                 angle_increment, scans_per_stream, sample_duration_us=31, stream=None, chunk_bytes=None,
                 chunk_rx_us=None, timing: "Timing | None" = None, scan_begin_ts_us=None):
        """Device addresses (the layouts of push), asynchronous on `stream` (None: the context's stream).  With
        chunk_bytes, chunk_rx_us, timing and scan_begin_ts_us, a stamped push."""
        if chunk_bytes is None and chunk_rx_us is None and timing is None and scan_begin_ts_us is None:
            self._ctx._check(self._L.rpl_capsule_stream_push_bytes_dev(
                self._h, _p(stream_bytes), _p(byte_counts), sample_duration_us, C.byref(params), _p(ranges),
                _p(intensities), _p(beam_counts), _p(angle_increment), _p(scans_per_stream), _p(stream)))
            return
        self._ctx._check(self._L.rpl_capsule_stream_push_bytes_ts_dev(
            self._h, _p(stream_bytes), _p(byte_counts), C.byref(timing) if timing is not None else None,
            chunk_bytes or 0, _p(chunk_rx_us), C.byref(params), _p(ranges), _p(intensities), _p(beam_counts),
            _p(angle_increment), _p(scans_per_stream), _p(scan_begin_ts_us), _p(stream)))

    def state(self):
        """(open_nodes, held_capsule, held_bytes)"""
        open_nodes, held, held_bytes = (np.zeros(self.n_streams, np.uint32) for _ in range(3))
        self._ctx._check(self._fn("state")(self._h, _p(open_nodes), _p(held), _p(held_bytes)))
        return open_nodes, held, held_bytes


class NormalStreamSession(CapsuleByteStreamSession):
    """The byte session on raw 0x81 standard-node byte streams, whose decoder takes no sample duration.  state()
    returns (open_nodes, held_bytes), held_bytes = bytes of the unfinished record held for the next push (0..4)."""

    def __init__(self, ctx: Context, n_streams: int, stride_bytes: int, max_nodes: int, max_scans: int):
        super().__init__(ctx, 0x81, n_streams, stride_bytes, max_nodes, max_scans)

    def push(self, stream_bytes, byte_counts, params: ScanParams, out=None, chunk_bytes=None, chunk_rx_us=None,
             timing: "Timing | None" = None):
        return super().push(stream_bytes, byte_counts, params, 0, out, chunk_bytes, chunk_rx_us, timing)

    def push_dev(self, stream_bytes, byte_counts, params: ScanParams, ranges, intensities, beam_counts,
                 angle_increment, scans_per_stream, stream=None, chunk_bytes=None, chunk_rx_us=None,
                 timing: "Timing | None" = None, scan_begin_ts_us=None):
        super().push_dev(stream_bytes, byte_counts, params, ranges, intensities, beam_counts, angle_increment,
                         scans_per_stream, 0, stream, chunk_bytes, chunk_rx_us, timing, scan_begin_ts_us)

    def state(self):
        """(open_nodes, held_bytes)"""
        open_nodes, held_bytes = (np.zeros(self.n_streams, np.uint32) for _ in range(2))
        self._ctx._check(self._fn("state")(self._h, _p(open_nodes), None, _p(held_bytes)))
        return open_nodes, held_bytes


class MixedByteStreamSession(CapsuleByteStreamSession):
    """A byte session in which every stream has its own answer type (rpl_capsule_stream_create_bytes_mixed): ans_types
    [n_streams], each 0x81..0x86, switched between pushes by set_answer_types.  Pushes, state and every other call are
    the byte session's; a push's sample_duration_us serves the capsule-type streams and is ignored for 0x81 ones."""

    def __init__(self, ctx: Context, ans_types, stride_bytes: int, max_nodes: int, max_scans: int):
        t = np.ascontiguousarray(ans_types, dtype=np.uint32)
        self._init(ctx, 0, t.size, 0, max_nodes, max_scans,
                   lambda h: ctx._L.rpl_capsule_stream_create_bytes_mixed(ctx._h, _p(t), t.size, stride_bytes,
                                                                           max_nodes, max_scans, C.byref(h)))
        self.stride_bytes = stride_bytes
        self.ans_types = t.copy()

    def set_answer_types(self, ans_types, mask=None):
        """The masked streams (mask [n_streams] of bool, None: all) take ans_types[s]; a stream whose type changes is
        reset as reset() resets it, the others are left alone."""
        t = np.ascontiguousarray(ans_types, dtype=np.uint32)
        assert t.shape == (self.n_streams,)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        assert m is None or m.shape == (self.n_streams,)
        self._ctx._check(self._fn("set_answer_types")(self._h, _p(t), _p(m)))
        sel = np.ones(self.n_streams, bool) if m is None else m.astype(bool)
        self.ans_types = np.where(sel, t, self.ans_types)


EXCHANGE_NCCL, EXCHANGE_COPY = 0, 1


def exchange_unique_id() -> bytes:
    """rank 0: a fresh NCCL unique id (128 bytes) for rpl_exchange_create on every rank."""
    buf = np.zeros(128, np.uint8)
    rc = lib().rpl_exchange_unique_id(_p(buf))
    if rc != RESULT_OK:
        raise RplError(rc, "rpl_exchange_unique_id failed (is libnccl.so.2 loadable?)")
    return buf.tobytes()


class Exchange:
    """rpl_exchange wrapper: the C++ all-gather of the fused cloud (include/rpl_b200.h)."""

    def __init__(self, ctx: "Context", unique_id, world: int, rank: int, slot_points: int, flags: int = 0):
        self._L, self._ctx = ctx._L, ctx
        idbuf = np.frombuffer(unique_id, np.uint8).copy() if unique_id is not None else None
        h = C.c_void_p()
        ctx._check(self._L.rpl_exchange_create(ctx._h, _p(idbuf), world, rank, slot_points, flags, C.byref(h)))
        self._h, self.world, self.rank, self.slot_points = h, world, rank, slot_points

    def allgather(self, xyzi, point_counts, n_scans, stride, mode=EXCHANGE_NCCL, stream=None) -> int:
        idx = C.c_uint32(0)
        self._ctx._check(self._L.rpl_exchange_allgather(self._h, _p(xyzi), _p(point_counts), n_scans, stride, mode,
                                                        _p(stream), C.byref(idx)))
        return idx.value

    def wait(self, index: int, stream=None):
        self._ctx._check(self._L.rpl_exchange_wait(self._h, index, _p(stream)))

    def release(self, index: int, stream=None):
        self._ctx._check(self._L.rpl_exchange_release(self._h, index, _p(stream)))

    def slot(self, index: int, rank: int):
        """(device address of the points, device address of the uint32 count) of one rank's slot."""
        pts, cnt = C.c_void_p(), C.c_void_p()
        self._ctx._check(self._L.rpl_exchange_slot(self._h, index, rank, C.byref(pts), C.byref(cnt)))
        return int(pts.value), int(cnt.value)

    def synchronize(self):
        self._ctx._check(self._L.rpl_exchange_synchronize(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._L.rpl_exchange_destroy(self._h)
            self._h = None


def host_alloc(nbytes: int) -> np.ndarray:
    """Pinned host memory as a uint8 numpy array (kept alive by a finalizer)."""
    L = lib()
    p = C.c_void_p()
    rc = L.rpl_host_alloc(nbytes, C.byref(p))
    if rc != RESULT_OK:
        raise RplError(rc, "rpl_host_alloc failed")
    buf = (C.c_uint8 * max(nbytes, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=np.uint8, count=nbytes)
    import weakref

    weakref.finalize(buf, L.rpl_host_free, p)
    return arr
