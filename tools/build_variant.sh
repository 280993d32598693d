#!/bin/bash
# usage: tools/build_variant.sh <tag> <unit: f16|f32|bf16|u8> [-DNAME=VALUE ...]
# Recompiles ONE dtype translation unit with extra defines and links it with the stock objects into
# comfyui-vrgamedevgirl_b200/lib/variants/libvrgdg_b200_<tag>.so (tuning experiments; select with VRGDG_B200_LIB=<path>).
set -e
tag=$1; unit=$2; shift 2
root=$(cd "$(dirname "$0")/.." && pwd)
pkg=$root/comfyui-vrgamedevgirl_b200
mkdir -p $pkg/lib/variants /tmp/vrgdg_var_$tag
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -Xfatbin -compress-all -I $root/include "$@" \
  -c $pkg/csrc/vrgdg_$unit.cu -o /tmp/vrgdg_var_$tag/vrgdg_$unit.o
objs=""
for u in abi f32 f16 bf16 u8; do
  if [ $u == $unit ]; then objs="$objs /tmp/vrgdg_var_$tag/vrgdg_$u.o"; else objs="$objs $pkg/build/vrgdg_$u.o"; fi
done
nvcc -shared -o $pkg/lib/variants/libvrgdg_b200_$tag.so $objs -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -lcudart_static -lpthread -ldl -lrt
echo built $pkg/lib/variants/libvrgdg_b200_$tag.so
