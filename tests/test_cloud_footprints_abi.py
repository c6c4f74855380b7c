"""The C ABI of footprints in the clouds: RPL_CLOUD_PER_STREAM_FOOTPRINTS and rpl_cloud_footprint_batch_dev, in the
header, the binding and the library's exports.  The refusals that need a device are in test_gpu_cloud_footprints.py."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    if not os.path.exists(R.capi.LIB_PATH):
        R.build()
    return R


def header():
    return open(os.path.join(ROOT, "include", "rpl_b200.h")).read()


def test_flag_value_is_the_headers_and_distinct():
    h = header()
    m = re.search(r"#define RPL_CLOUD_PER_STREAM_FOOTPRINTS (\d+)u", h)
    assert m and int(m.group(1)) == 8
    others = [int(v) for v in re.findall(r"#define RPL_CLOUD_\w+ (\d+)u", h)]
    assert sorted(others) == [1, 2, 4, 8]


def test_binding_and_exports(R):
    assert R.CLOUD_PER_STREAM_FOOTPRINTS == 8
    assert "rpl_cloud_footprint_batch_dev" in R.capi.EXPORTS
    assert hasattr(ctypes.CDLL(R.capi.LIB_PATH), "rpl_cloud_footprint_batch_dev")
    assert hasattr(R.Context, "cloud_footprint_batch_dev")
    src = re.sub(r"/\*.*?\*/", "", header(), flags=re.S)
    decl = re.search(r"rpl_result rpl_cloud_footprint_batch_dev\(([^)]*)\)", src).group(1)
    assert "const rpl_scan_footprint* footprint" in decl
    argtypes = R.lib().rpl_cloud_footprint_batch_dev.argtypes
    assert len(argtypes) == decl.count(",") + 1 == 10
