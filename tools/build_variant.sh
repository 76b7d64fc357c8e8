#!/bin/bash
# tools/build_variant.sh <tag> <extra nvcc flags for resample.cu...>  ->  timg_b200/libb200timg_<tag>.so (tuning builds,
# loaded with B200TIMG_LIBFILE=...; everything but resample.cu is taken from the regular build's objects)
set -e
cd "$(dirname "$0")/../timg_b200/csrc"
tag=$1; shift
NV="/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-ffp-contract=off -I../../include"
$NV "$@" -c resample.cu -o /tmp/resample_$tag.o -Xptxas -v 2> /tmp/resample_$tag.log
objs=$(ls *.o | grep -v '^resample\.o$' | tr '\n' ' ')
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../libb200timg_$tag.so $objs /tmp/resample_$tag.o -cudart static
grep -A2 "resample_v3_kernelILi6ELi6EEv" /tmp/resample_$tag.log | grep -E "Used|spill" 
