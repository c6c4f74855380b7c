"""CPU-side checks of the stream-record C-ABI: the header declares rpl_capsule_stream_export and _import and the record
version, and the ctypes binding's argtypes are those declarations."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
CTYPE = {"rpl_capsule_stream*": C.c_void_p, "const uint32_t*": C.c_void_p, "uint32_t": C.c_uint32,
         "uint8_t*": C.c_void_p, "const uint8_t*": C.c_void_p, "uint64_t": C.c_uint64, "uint64_t*": C.c_void_p,
         "const uint64_t*": C.c_void_p}


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _params(name):
    m = re.search(r"rpl_result\s+" + name + r"\s*\((.*?)\)\s*;", _header(), re.S)
    assert m, name
    return [re.sub(r"\s*\*\s*", "* ", p.strip()).rsplit(" ", 1)[0].replace("* ", "*").strip() for p in m.group(1).split(",")]


def test_header_declares_both_calls_and_the_version():
    assert _params("rpl_capsule_stream_export") == ["rpl_capsule_stream*", "const uint32_t*", "uint32_t", "uint8_t*",
                                                   "uint64_t", "uint64_t*", "uint64_t*"]
    assert _params("rpl_capsule_stream_import") == ["rpl_capsule_stream*", "const uint32_t*", "uint32_t",
                                                   "const uint8_t*", "const uint64_t*", "uint64_t"]
    assert int(re.search(r"#define\s+RPL_STREAM_RECORD_VERSION\s+(\d+)u", _header()).group(1)) == 1


@pytest.mark.parametrize("name", ["rpl_capsule_stream_export", "rpl_capsule_stream_import"])
def test_binding_argtypes_are_the_declaration(name):
    import rplidar_ros2_driver_b200 as R

    if not os.path.exists(R.capi.LIB_PATH):
        R.build()
    fn = getattr(R.lib(), name)
    assert name in R.capi.EXPORTS
    assert list(fn.argtypes) == [CTYPE[p] for p in _params(name)]
    assert fn.restype == C.c_uint32
