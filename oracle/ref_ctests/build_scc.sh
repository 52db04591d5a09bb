#!/bin/bash
# TEST INFRASTRUCTURE: compile the reference's OWN C-API test for strongly connected components —
# cpp/tests/c_api/strongly_connected_components_test.c, unmodified, from where it lies under $REF — against this
# repository's headers, with the same support code and flags as build.sh, and link it with a libcugraph_c build (default:
# the CPU emulation build; pass the CUDA library to get a binary for a GPU machine).  Output only into oracle/_ref/
# (git-ignored).  No reference source is copied.
#   bash oracle/ref_ctests/build_scc.sh [path/to/libcugraph_c*.so] [suffix of the binary]
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
REF="${REF:-/root/reference}"
LIB="${1:-$ROOT/cugraph_b200/lib/libcugraph_c_emu.so}"
SUFFIX="${2:-}"
OUT="$ROOT/oracle/_ref"
CUDA_INC="${CUDA_INC:-/usr/local/cuda/include}"
[ -f "$REF/cpp/tests/c_api/strongly_connected_components_test.c" ] || { echo "reference sources not found under $REF"; exit 3; }
[ -f "$LIB" ] || { echo "library $LIB not built"; exit 4; }
mkdir -p "$OUT"
LIBDIR="$(dirname "$LIB")"; LIBNAME="$(basename "$LIB")"
gcc -std=gnu11 -O1 -w -I "$ROOT/include" -I "$HERE/include" -I "$CUDA_INC" \
    "$REF/cpp/tests/c_api/strongly_connected_components_test.c" "$HERE/support.c" \
    -o "$OUT/ref_strongly_connected_components_test${SUFFIX}" \
    -L "$LIBDIR" -l:"$LIBNAME" -Wl,-rpath,'$ORIGIN/../../cugraph_b200/lib' -Wl,-rpath,"$LIBDIR" -lm
echo "built: $OUT/ref_strongly_connected_components_test${SUFFIX} (against $LIB)"
