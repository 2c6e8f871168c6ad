#!/usr/bin/env bash
# Build libpinb200.so (sm_90a, H100) in-tree: every .cu is compiled to build/<name>.o when it (or any header) is newer,
# then linked.  Usage: build.sh [extra nvcc flags]   (extra flags force a full rebuild)
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
out="$here/../libpinb200.so"
obj="$here/build"
mkdir -p "$obj"
[ $# -gt 0 ] && rm -f "$obj"/*.o
newest_hdr=$(ls -t "$here"/*.cuh "$here"/../../include/pinb200.h | head -1)
log="$here/../build.log"
: > "$log"
pids=()
for src in "$here"/*.cu; do
  o="$obj/$(basename "${src%.cu}").o"
  if [ ! -f "$o" ] || [ "$src" -nt "$o" ] || [ "$newest_hdr" -nt "$o" ]; then
    ( nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v "$@" \
           -c -o "$o" "$src" > "$o.log" 2>&1 || { cat "$o.log"; rm -f "$o"; exit 1; } ) &
    pids+=($!)
  fi
done
fail=0
for p in "${pids[@]:-}"; do [ -n "$p" ] && { wait "$p" || fail=1; }; done
cat "$obj"/*.o.log >> "$log" 2>/dev/null || true
[ $fail -eq 0 ] || { grep -E "error" "$log" | head -40; exit 1; }
nvcc -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fPIC -o "$out" "$obj"/*.o
grep -E "error|warning: v|spill|Used" "$log" | grep -vE "^$" | tail -${PINB_BUILD_TAIL:-12} || true
echo "built $out"
