#!/bin/bash
# ThreadSanitizer over the CUDA-on-CPU shim build of the kernels (CPU only; see tests/tools/emu_race_check.py).
set -e
cd "$(dirname "$0")/../.."
python tests/cuda_emu/build.py > /dev/null
( cd tests/cuda_emu && g++ -std=c++20 -O1 -g -pthread -fPIC -shared -fsanitize=thread -ffp-contract=off -Wno-unknown-pragmas -Wno-attributes \
    -DPOSE_MIXED_SOLVE=1 -I. -Ibuild -o build/libcuda_emu_tsan.so emu_entry.cpp emu_runtime.cpp build/host_tables.cpp build/quadtree_host.cpp )
for a in extract dilate; do
    echo "== $a"
    LD_PRELOAD=$(g++ -print-file-name=libtsan.so) TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0" python tests/tools/emu_race_check.py $a 2>&1 \
        | grep -E "^(extract|dilate) |WARNING: ThreadSanitizer|    #0 " | sort | uniq -c | sort -rn | head -8
done
