#!/bin/bash
# Memory-safety pass over the emulated library: build it with AddressSanitizer and run the emulation tests + the fuzzer.
# "Device" memory is malloc'ed host memory in the emulation, so an out-of-bounds access of a kernel is a heap error here.
#   bash emu/run_asan.sh [fuzz seconds]
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd); CSRC=$ROOT/cugraph_b200/csrc; OUT=/tmp/libcugraph_c_emu_asan.so
SRCS=""; for f in capi_basic.cu capi_graph.cu graph_build.cu sweep_layout.cu sweep.cu pagerank.cu traverse.cu mg.cu; do SRCS="$SRCS -x c++ $CSRC/$f"; done
/usr/bin/g++ -std=c++17 -O1 -g -fPIC -shared -fvisibility=hidden -DB200_HOST_EMU -fsanitize=address -fno-omit-frame-pointer \
  -I $ROOT/emu -I $ROOT/include -I $CSRC -Wno-attributes $SRCS -x c++ $ROOT/emu/emu_debug.cpp -o $OUT
# libstdc++ too: Python does not link it, and ASan resolves its __cxa_throw interceptor when it starts
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libstdc++.so)"
export ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1
cd $ROOT
python - <<PY
import sys
sys.path.insert(0, "$ROOT"); sys.path.insert(0, "$ROOT/emu")
import build_emu
build_emu.build = lambda force=False: "$OUT"
import pytest
sys.exit(pytest.main(["-x", "-q", "-p", "no:cacheprovider", "tests/test_emu_staging_cpu.py", "tests/test_sweep_bands_cpu.py", "tests/test_emu_algorithms_cpu.py", "tests/test_emu_mg_cpu.py", "tests/test_emu_goldens_cpu.py", "tests/test_emu_edge_cases_cpu.py"]))
PY
python emu/fuzz.py ${1:-120} $OUT
