#!/bin/bash
# Builds variant_bench and one cubin per leaf-hash variant into tools/variants/out/ (git-ignored).
set -e
cd "$(dirname "$0")"
mkdir -p out
NV="nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo"
nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -o out/variant_bench variant_bench.cu -lcuda
v() { name=$1; shift; $NV -cubin -o out/$name.cubin leaf_kernel.cu "$@" & }
v base
v cvtmagic -DGL_CVT_MAGIC
v pfast -DGL_PARTIAL_FAST
v mdsint -DGL_MDS_INT
v mulx -DGL_MUL_EXPLICIT
v sqr3 -DGL_SQR_3WIDE
v sboxsqr4 -DGL_SBOX_SQR4
v sboxi2f -DGL_SBOX_I2F
v movehand -DGL_SBOX_MOVE_HANDOVER                     # the S-box limbs from register-built doubles and 5 DADDs
v retr96 -DGL_RET_REDUCE96                             # the FP64 -> u64 return through a 96-bit reduction
v prevbase -DGL_SBOX_MOVE_HANDOVER -DGL_RET_REDUCE96   # both: the full round before the integer hand-overs
v pairf64 -DGL_PAIR_RENORM_F64                          # the partial-round pair before the ALU renormalisation
v parent -DGL_SBOX_SQR4 -DGL_SBOX_I2F -DVB_MINB=5      # the S-box and budget before the spill-free change
v parentb4 -DGL_SBOX_SQR4 -DGL_SBOX_I2F                # that S-box at the shipped budget
v redv1 -DGL_REDUCE_V1
v nosync -DVB_SYNC=0
v t128b5 -DVB_MINB=5
v t128b6 -DVB_MINB=6
v t256b2 -DVB_THREADS=256 -DVB_MINB=2
v t64b10 -DVB_THREADS=64 -DVB_MINB=10
wait
for x in "$@"; do :; done
ls out/*.cubin | wc -l
