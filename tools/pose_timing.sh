#!/bin/bash
# Development aid (needs a GPU): rebuild pose_kernels.o with -DPOSE_TIMING (clock64 per phase, printed by rank 0 of the cluster, with the
# number of build passes, evaluated / accepted trials and skipped repeat rounds of each call), run a short chain, restore the normal object.
set -e
cd orb_slam3_rgbl_b200/csrc
F="-gencode arch=compute_90a,code=sm_90a --extended-lambda -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-ffp-contract=off -fmad=true"
cp obj/pose_kernels.o /tmp/pose_kernels.o.keep; cp ../librgbl_b200.so /tmp/librgbl_b200.so.keep
nvcc $F -DPOSE_TIMING -c -o obj/pose_kernels.o pose_kernels.cu && nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../librgbl_b200.so obj/*.o
cd ../..
python tools/run_chain_once.py 5 2>&1 | grep "pose n=" | tail -8
cp /tmp/pose_kernels.o.keep orb_slam3_rgbl_b200/csrc/obj/pose_kernels.o; cp /tmp/librgbl_b200.so.keep orb_slam3_rgbl_b200/librgbl_b200.so
