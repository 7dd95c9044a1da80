# usage: bash scripts/host_sanitize.sh  (CPU only) -- the product's host state machine under AddressSanitizer + UBSan:
# tests/cpp/host_harness.cpp (= csrc/estimator.h + estimator_host.cpp.inc + tracker_host.cpp.inc + triangulate.h + homography.h) is
# compiled with -fsanitize=address,undefined and driven by the host-logic and twin tests (whole point-cloud and tracker-only image
# sequences, every decision checked against the oracle).
set -e
SO=/tmp/libhost_harness_asan.so
g++ -std=c++17 -O1 -g -march=x86-64-v3 -fsanitize=address,undefined -fno-omit-frame-pointer -I "${CUDA_HOME:-/usr/local/cuda}/include" -shared -fPIC tests/cpp/host_harness.cpp -o $SO
# libstdc++ has to be preloaded next to libasan, otherwise ASan's __cxa_throw interceptor finds no real function inside a Python process
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libstdc++.so.6)" ASAN_OPTIONS=detect_leaks=0 XIVO_HH_SO=$SO
python -m pytest tests/test_host_logic.py tests/test_host_twin.py -q -p no:cacheprovider 2>&1 | tee /tmp/host_sanitize.log | tail -3
! grep -q "runtime error\|AddressSanitizer" /tmp/host_sanitize.log && echo "sanitizers: no report"
