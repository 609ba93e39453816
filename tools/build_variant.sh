#!/bin/bash
# usage: tools/build_variant.sh <name> <parse_kernels.cuh to use> [extra nvcc flags...]
# builds csvplus_b200/_var/<name>.so = the current library with parse.cu compiled against the given kernel header
set -e
name=$1; hdr=$2; shift 2
root=$(cd "$(dirname "$0")/.." && pwd)
tmp=$(mktemp -d)
mkdir -p $tmp/csvplus_b200 $tmp/include
cp -r $root/csvplus_b200/csrc $tmp/csvplus_b200/csrc
cp $root/include/csvplus_b200.h $tmp/include/
cp "$hdr" $tmp/csvplus_b200/csrc/parse_kernels.cuh
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr --extended-lambda "$@" -c $tmp/csvplus_b200/csrc/parse.cu -o $tmp/parse.o
objs=$(ls $root/csvplus_b200/_obj/*.o | grep -v '/parse.o')
mkdir -p $root/csvplus_b200/_var
/usr/local/cuda/bin/nvcc -shared -cudart static -o $root/csvplus_b200/_var/$name.so $tmp/parse.o $objs -ldl
rm -rf $tmp
echo built $root/csvplus_b200/_var/$name.so
