#!/bin/bash
# usage: tools/build_variant.sh <name> [git-rev | -] [replacement decode_mega.cu]
# Builds a complete alternative libdtk into variants/libdtk_<name>.so (git-ignored) for same-machine A/B
# runs through DTK_B200_LIB. Sources: the working tree ("-") or a git revision; optionally one decode_mega.cu swapped in.
set -e
name=$1; rev=${2:--}; swap=$3
root=$(cd "$(dirname "$0")/.." && pwd)
tmp=$(mktemp -d /tmp/dtkvar.XXXX)
mkdir -p "$tmp/detikzify_b200"
if [ "$rev" = "-" ]; then
  cp -r "$root/detikzify_b200/csrc" "$tmp/detikzify_b200/csrc"; cp -r "$root/include" "$tmp/include"
  rm -rf "$tmp/detikzify_b200/csrc/build" "$tmp/detikzify_b200/csrc"/*.so
else
  (cd "$root" && git archive "$rev" detikzify_b200/csrc include | tar -x -C "$tmp")
fi
[ -n "$swap" ] && cp "$swap" "$tmp/detikzify_b200/csrc/decode_mega.cu"
mkdir -p "$root/variants"
cd "$tmp/detikzify_b200/csrc"
pids=()
for f in *.cu; do
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -I "$tmp/include" -c "$f" -o "${f%.cu}.o" > "${f%.cu}.log" 2>&1 &
  pids+=($!)
done
for p in "${pids[@]}"; do wait "$p" || { cat *.log | grep -i error; echo "compile failed"; exit 1; }; done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o "$root/variants/libdtk_$name.so" *.o
echo "built variants/libdtk_$name.so ($(nm -D "$root/variants/libdtk_$name.so" | grep -c ' T dtk_') exported dtk_ symbols)"
rm -rf "$tmp"
