#!/usr/bin/env bash
# Builds librplidar_b200.so in-tree for sm_90a (H100).  nvcc cross-compiles without a GPU.
# Every csrc/*.cu is compiled to its own object (in parallel, only when stale) and linked.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
OUT="${RPL_OUT:-$HERE/librplidar_b200.so}"
OBJ="${RPL_OBJ:-$HERE/build}"
mkdir -p "$OBJ"
SRCS=("$HERE"/csrc/*.cu)
CFLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo --fmad=false \
        -Xcompiler -fPIC,-O2,-ffp-contract=off,-Wall,-Wno-address-of-packed-member)
if [[ "${RPL_PTXAS_V:-0}" == "1" ]]; then CFLAGS+=(-Xptxas -v); fi
# a change of flags or of any header rebuilds everything
STAMP="$OBJ/.flags"
NEWEST_HDR=$(ls -t "$HERE"/csrc/*.h "$HERE"/csrc/*.cuh "$HERE"/../include/*.h | head -1)
if [[ ! -f "$STAMP" || "$(cat "$STAMP")" != "${CFLAGS[*]}" ]]; then rm -f "$OBJ"/*.o; echo "${CFLAGS[*]}" > "$STAMP"; fi
pids=()
objs=()
for s in "${SRCS[@]}"; do
  o="$OBJ/$(basename "${s%.cu}").o"
  objs+=("$o")
  # decode_list.cu compiles decode_formats.cu a second time (its stream-list instantiations)
  dep="$s"; [[ "$(basename "$s")" == decode_list.cu ]] && dep="$HERE/csrc/decode_formats.cu"
  if [[ ! -f "$o" || "$s" -nt "$o" || "$dep" -nt "$o" || "$NEWEST_HDR" -nt "$o" ]]; then
    ( "$NVCC" "${CFLAGS[@]}" -c -o "$o.tmp" "$s" && mv "$o.tmp" "$o" ) &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]:-}"; do
  if [[ -n "$p" ]]; then wait "$p" || rc=1; fi
done
if [[ $rc -ne 0 ]]; then echo "compile failed" >&2; exit 1; fi
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared -cudart shared -o "$OUT" "${objs[@]}" -ldl
echo "built $OUT"
