#!/bin/bash
# Link test for the C++ drop-in (SURVEY.md section 8b): compile the reference's UNMODIFIED sd.cpp, llm.cpp and exports.cpp
# where they lie under $REF against the reference's own onnxstream.h, and link them with compat_onnxstream.cpp + the
# engine instead of the reference's onnxstream.cpp.  Outputs go to oracle/_ref/link_test/ (git-ignored; they travel with the oracle and
# find the engine library through an rpath relative to themselves).  Nothing is copied.
set -euo pipefail
REF=${REF:?set REF to the src directory of the reference checkout}
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=$ROOT/oracle/_ref/link_test
TORCH=$(python3 -c "import torch,os;print(os.path.dirname(torch.__file__))")
CXX=${CXX_BIN:-/usr/bin/g++}
mkdir -p "$OUT"
cat > "$OUT/cpuinfo_stub.c" <<'EOC'
/* sd.cpp only asks cpuinfo whether fp16 arithmetic is available on the host CPU (src/sd.cpp:198-199); the engine
   does not care, so report "no" like a CPU without the extension would. */
#include <stdbool.h>
struct cpuinfo_x86_isa { int unused; };
bool cpuinfo_initialize(void) { return true; }
struct cpuinfo_x86_isa cpuinfo_isa = { 0 };
EOC
gcc -c "$OUT/cpuinfo_stub.c" -o "$OUT/cpuinfo_stub.o"
FLAGS="-std=c++20 -O1 -fPIC -fcoroutines -I$REF -I$TORCH/include -I/usr/local/cuda/include"
# compat.o depends on the engine headers: always rebuilt (a stale one is an ABI mismatch against libonnxstream_b200.so);
# the reference's own translation units only change with the reference, so they are compiled once.
$CXX $FLAGS -c "$ROOT/onnxstream_b200/csrc/compat_onnxstream.cpp" -I"$ROOT/onnxstream_b200/csrc" -o "$OUT/compat.o"
[ "$OUT/sd.o" -nt "$REF/sd.cpp" ] || $CXX $FLAGS -c "$REF/sd.cpp" -o "$OUT/sd.o"
[ "$OUT/llm.o" -nt "$REF/llm.cpp" ] || $CXX $FLAGS -c "$REF/llm.cpp" -o "$OUT/llm.o" 2>/dev/null
[ "$OUT/exports.o" -nt "$REF/exports.cpp" ] || $CXX $FLAGS -c "$REF/exports.cpp" -o "$OUT/exports.o"
LIB="$ROOT/onnxstream_b200/csrc/libonnxstream_b200.so"
RPATH='$ORIGIN/../../../onnxstream_b200/csrc'      # oracle/_ref/link_test -> the engine library of the same tree
$CXX -o "$OUT/sd" "$OUT/sd.o" "$OUT/compat.o" "$OUT/cpuinfo_stub.o" -L"$(dirname $LIB)" -lonnxstream_b200 -Wl,-rpath,"$RPATH" -lpthread
$CXX -o "$OUT/llm" "$OUT/llm.o" "$OUT/compat.o" -L"$(dirname $LIB)" -lonnxstream_b200 -Wl,-rpath,"$RPATH" -lpthread
$CXX -shared -o "$OUT/libonnxstream_ref_exports.so" "$OUT/exports.o" "$OUT/compat.o" -L"$(dirname $LIB)" -lonnxstream_b200 -Wl,-rpath,"$RPATH" -lpthread
echo "undefined onnxstream:: symbols required by the apps:"
nm -uC "$OUT/sd.o" "$OUT/llm.o" "$OUT/exports.o" | grep "onnxstream::" | sed 's/^ *U //' | sort -u
echo "linked: $OUT/sd $OUT/llm $OUT/libonnxstream_ref_exports.so"
