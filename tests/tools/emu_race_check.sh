#!/bin/bash
# ThreadSanitizer over the emulated library built with -fsanitize=thread (CPU only; see tests/tools/emu_race_check.py).
set -e
cd "$(dirname "$0")/../.."
python tests/cuda_emu/build.py thread > /dev/null
for a in extract dilate; do
    echo "== $a"
    LD_PRELOAD=$(g++ -print-file-name=libtsan.so) TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0" python tests/tools/emu_race_check.py $a 2>&1 \
        | grep -E "^(extract|dilate) |WARNING: ThreadSanitizer|    #0 " | sort | uniq -c | sort -rn | head -8
done
