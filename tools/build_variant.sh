#!/bin/bash
# usage: [SOURCES="join.cu gather.cu"] tools/build_variant.sh <name> <parse_kernels.cuh to use, or - for the current one> [extra nvcc flags...]
# builds csvplus_b200/_var/<name>.so = the current library with the SOURCES (default parse.cu) recompiled with the extra
# flags, parse.cu against the given kernel header; e.g. the -D diagnostic switches of rowhash_scatter / rowhash_probe:
#   SOURCES="join.cu gather.cu" tools/build_variant.sh scatter_no_atomic - -DRH_DIAG_NO_ATOMIC
set -e
name=$1; hdr=$2; shift 2
srcs=${SOURCES:-parse.cu}
root=$(cd "$(dirname "$0")/.." && pwd)
tmp=$(mktemp -d)
mkdir -p $tmp/csvplus_b200 $tmp/include
cp -r $root/csvplus_b200/csrc $tmp/csvplus_b200/csrc
cp $root/include/csvplus_b200.h $tmp/include/
[ "$hdr" = - ] || cp "$hdr" $tmp/csvplus_b200/csrc/parse_kernels.cuh
objs=$(ls $root/csvplus_b200/_obj/*.o)
for s in $srcs; do
    /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr --extended-lambda -I $root/csvplus_b200/_obj "$@" -c $tmp/csvplus_b200/csrc/$s -o $tmp/${s%.cu}.o
    objs=$(echo "$objs" | grep -v "/${s%.cu}.o$")
done
mkdir -p $root/csvplus_b200/_var
/usr/local/cuda/bin/nvcc -shared -cudart static -o $root/csvplus_b200/_var/$name.so $tmp/*.o $objs -ldl
rm -rf $tmp
echo built $root/csvplus_b200/_var/$name.so
