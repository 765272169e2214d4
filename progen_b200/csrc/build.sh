#!/usr/bin/env bash
# Build libprogen_b200.so in-tree for sm_90a (H100) (cross-compiles without a GPU).  Usage: build.sh [-j N]
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/../libprogen_b200.so"
OBJ="$HERE/build"
mkdir -p "$OBJ"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O3
       --expt-relaxed-constexpr -DCUDA_VERSION_STR="\"12.9\"" -I"$HERE" -I"$HERE/../../include")
SRCS=(api gemm_tc gemm_simt elementwise ln_stream attn_simt attn_wgmma optim decode_persist)
pids=()
for s in "${SRCS[@]}"; do
  [ -f "$HERE/$s.cu" ] || continue
  if [ ! -f "$OBJ/$s.o" ] || [ "$HERE/$s.cu" -nt "$OBJ/$s.o" ] || [ -n "$(find "$HERE" "$HERE/../../include" -maxdepth 1 \( -name '*.cuh' -o -name '*.h' \) -newer "$OBJ/$s.o" 2>/dev/null)" ]; then
    "$NVCC" "${FLAGS[@]}" -c "$HERE/$s.cu" -o "$OBJ/$s.o" &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
objs=()
for s in "${SRCS[@]}"; do [ -f "$OBJ/$s.o" ] && objs+=("$OBJ/$s.o"); done
"$NVCC" -shared -o "$OUT" "${objs[@]}" -cudart static -Xlinker --no-undefined
echo "built $OUT"
