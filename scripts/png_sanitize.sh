# usage: bash scripts/png_sanitize.sh  (CPU only) -- the PNG decoder of xivo_b200/csrc/png.cuh under AddressSanitizer + UBSan:
# tests/cpp/png_harness.cpp is compiled with -fsanitize=address,undefined and driven by the harness tests of tests/test_png_logic.py
# (corpus against the oracle, the corrupt deflate set, every truncation, random bit flips).
set -e -o pipefail
D="${PNG_SAN_DIR:-/tmp}"
SO="$D/libpng_harness_asan.so"
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-sanitize-recover=undefined -fno-omit-frame-pointer -shared -fPIC tests/cpp/png_harness.cpp -o "$SO"
# libstdc++ has to be preloaded next to libasan, otherwise ASan's __cxa_throw interceptor finds no real function inside a Python process
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libstdc++.so.6)" ASAN_OPTIONS=detect_leaks=0 XIVO_PNG_HARNESS_SO="$SO"
python -m pytest tests/test_png_logic.py -q -p no:cacheprovider -k "harness and not sanitizers" 2>&1 | tee "$D/png_sanitize.log" | tail -3
! grep -q "runtime error\|AddressSanitizer" "$D/png_sanitize.log" && echo "sanitizers: no report"
