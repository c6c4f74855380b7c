"""rplidar_ros2_driver_b200 -- H100-native (sm_90a) per-scan point-processing hot path of
frozenreboot/rplidar_ros2_driver behind a C-ABI (include/rpl_b200.h).

  csrc/   hand-written sm_90a CUDA kernels + the C-ABI (librplidar_b200.so)
  host/   C++17 host mirror of the reference's LidarDriverInterface / publish_scan seam
  capi.py ctypes binding used by tests/ and bench.py

There is no CPU implementation here: the oracle lives under /oracle and is test-only.
"""
from .capi import (  # noqa: F401
    NODE_DTYPE, CapsuleByteStreamSession, CapsuleStreamSession, Context, DenseStreamSession, Exchange, MixedByteStreamSession,
    NormalStreamSession, RplError, exchange_unique_id, EXCHANGE_NCCL, EXCHANGE_COPY, Timing, build, cloud_params, host_alloc, lib, scan_params,
    LidarSettings, lidar_settings, PushInput, FLAG_PER_STREAM, CLOUD_PER_STREAM, CloudSettings, cloud_settings,
    CLOUD_PER_STREAM_CHAIN, CLOUD_PER_STREAM_FOOTPRINTS, FLAG_PER_STREAM_FILTERS, ScanFilterSettings, scan_filter_settings,
    ScanFootprint, scan_footprint, ScanCloudParams, scan_cloud_params, SCAN_CLOUD_INTENSITY, SCAN_CLOUD_INDEX,
    SCAN_CLOUD_DISTANCE, SCAN_CLOUD_TIMESTAMP, MsgsOut, ScanCloudTransform, scan_cloud_transform, SCAN_CLOUD_VIEWPOINT,
    SCAN_CLOUD_PER_STREAM_TRANSFORMS, RescanSettings, rescan_settings, rescan_ranges_size, RescanWindow, rescan_window,
    RESCAN_MERGE_NONE,
    FLAG_FORCE_GENERAL, FLAG_NO_TMA, FLAG_NO_SMALL, CLOUD_NO_FUSED, PATH_FAST, PATH_GENERAL, RESULT_OK, RESULT_OPERATION_FAIL, RESULT_INVALID_DATA,
)
