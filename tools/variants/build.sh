#!/bin/bash
cd "$(dirname "$0")"
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC -shared \
    -I ../../pypose_b200/csrc variants.cu -o libvariants.so
