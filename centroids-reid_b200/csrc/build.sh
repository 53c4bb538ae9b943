#!/usr/bin/env bash
# Builds libctl_b200.so (sm_90a only) next to the Python package.  nvcc cross-compiles
# without a GPU.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libctl_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall
       --expt-relaxed-constexpr -Xptxas -v)
mkdir -p "${HERE}/obj"
pids=()
for src in "${HERE}"/*.cu; do
  obj="${HERE}/obj/$(basename "${src%.cu}").o"
  if [[ ! -f "$obj" || "$src" -nt "$obj" || "${HERE}/wgmma.cuh" -nt "$obj" || "${HERE}/common.h" -nt "$obj" \
        || "${HERE}/resnet.h" -nt "$obj" || "${HERE}/../../include/ctl_b200.h" -nt "$obj" ]]; then
    ( "$NVCC" "${FLAGS[@]}" -c "$src" -o "$obj" > "${obj%.o}.log" 2>&1 || { cat "${obj%.o}.log"; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" "${HERE}"/obj/*.o -lcudart
echo "built $OUT"
