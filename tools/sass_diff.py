#!/usr/bin/env python3
"""Compares two builds of librplidar_b200.so (or of one object file) kernel by kernel: the SASS of every kernel in
OLD must be instruction for instruction the SASS of the kernel of the same name in NEW.  Kernels only NEW has are
listed as added.  Exit status 1 when a kernel of OLD is missing from NEW or compiles differently.

    git worktree add /tmp/parent HEAD~1 && bash /tmp/parent/rplidar_ros2_driver_b200/build.sh
    bash rplidar_ros2_driver_b200/build.sh
    python tools/sass_diff.py /tmp/parent/rplidar_ros2_driver_b200/librplidar_b200.so \\
        rplidar_ros2_driver_b200/librplidar_b200.so

Register and shared-memory figures come from the compiler: RPL_PTXAS_V=1 bash rplidar_ros2_driver_b200/build.sh.
"""
import argparse
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def kernels(path):
    """{function name: [instructions]} of every function in the file's sm_90a SASS (addresses and the line-info
    comments dropped, so that a kernel moved within the file still compares equal)"""
    txt = subprocess.run([CUOBJDUMP, "-sass", path], check=True, capture_output=True, text=True).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            # internal-linkage names carry two hashes, of the build and of the file's contents:
            # _GLOBAL__N__<hash>_<len>_<file>_cu_<hash>
            name = re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+_\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1", m.group(1))
            out[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)
        if name and m:
            out[name].append(m.group(1))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("old")
    ap.add_argument("new")
    args = ap.parse_args()
    old, new = kernels(args.old), kernels(args.new)
    bad = 0
    for k in sorted(old):
        if k not in new:
            print(f"MISSING  {k}")
            bad += 1
        elif old[k] != new[k]:
            print(f"CHANGED  {k} ({len(old[k])} -> {len(new[k])} instructions)")
            bad += 1
    for k in sorted(set(new) - set(old)):
        print(f"ADDED    {k} ({len(new[k])} instructions)")
    print(f"{len(old) - bad} of {len(old)} kernels of {args.old} unchanged")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
