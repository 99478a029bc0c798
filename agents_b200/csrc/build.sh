#!/usr/bin/env bash
# Builds agents_b200/lib/libb200rl.so for sm_90a (nvcc cross-compiles without a GPU).
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
out="$here/../lib"
mkdir -p "$out" "$here/obj"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC --split-compile=0
       --expt-relaxed-constexpr -Xptxas -v)
pids=()
for f in "$here"/*.cu; do
  o="$here/obj/$(basename "${f%.cu}").o"
  stale=0
  for dep in "$f" "$here"/*.cuh "$here/../../include/b200rl.h"; do
    [[ ! -f "$o" || "$dep" -nt "$o" ]] && stale=1
  done
  if [[ $stale -eq 1 ]]; then
    "$NVCC" "${FLAGS[@]}" -c "$f" -o "$o" > "$o.log" 2>&1 &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]:-}"; do
  [[ -z "$p" ]] && continue
  wait "$p" || rc=1
done
if [[ $rc -ne 0 ]]; then
  cat "$here"/obj/*.log | grep -E "error|Error" -A3 | head -80
  echo "BUILD FAILED" >&2
  rm -f "$out/libb200rl.so"   # never leave a stale library behind a failed build
  exit 1
fi
"$NVCC" -shared -gencode arch=compute_90a,code=sm_90a -o "$out/libb200rl.so" "$here"/obj/*.o -lcudart_static -ldl -lrt -lpthread
echo "built $out/libb200rl.so"
