#!/bin/bash
# Builds an alternative libzgpu (tuning experiments): scripts/build_variant.sh NAME "-DZG_PHASE_CLOCKS=1 ..."
# -> spicedb-kubeapi-proxy_b200/variants/libzgpu_NAME.so ; select it with ZGPU_LIB=<path>.
set -e
name=$1; flags=$2
root=$(cd "$(dirname "$0")/.." && pwd)
src=$root/spicedb-kubeapi-proxy_b200/csrc
out=$root/spicedb-kubeapi-proxy_b200/variants
tmp=$(mktemp -d)
mkdir -p $out
NV="/usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC --expt-relaxed-constexpr $flags"
for f in capi.cu device.cu build.cu; do $NV -c $src/$f -o $tmp/$f.o & done
for f in schema.cc store.cc listfilter.cc; do $NV -x cu -c $src/$f -o $tmp/$f.o & done
wait
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $out/libzgpu_$name.so $tmp/*.o -cudart static
rm -rf $tmp
echo built $out/libzgpu_$name.so
