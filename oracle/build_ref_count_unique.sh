#!/usr/bin/env bash
# Build the UNMODIFIED reference's count_unique (fbreitwieser/krakenuniq src/count_unique.cpp) from the sources under
# $KUQ_REFERENCE_SRC into oracle/_ref/count_unique (git-ignored), with the flags and command-line work-arounds of
# build_ref.sh beside it.  TEST INFRASTRUCTURE ONLY: tests/test_count_unique_cpu.py records its runs with it, and
# krakenuniq_b200/bench_count_unique.py times it when it exists; nothing under krakenuniq_b200/ links it.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
SRC="${KUQ_REFERENCE_SRC:-}"
OUT="$HERE/_ref"
if [ ! -d "$SRC" ]; then
  echo "build_ref_count_unique.sh: set KUQ_REFERENCE_SRC to the reference's src/ directory" >&2
  exit 3
fi
mkdir -p "$OUT/obj"
CXX="${KUQ_CXX:-/usr/bin/g++}"
CXXFLAGS=(-Wall -Wextra -Wfatal-errors -pipe -O2 -std=c++11 -fopenmp -DNDEBUG -w
          -include cstdint -I"$SRC" -I"$SRC/gzstream"
          -DBXZSTR_CONFIG_HPP -DBXZSTR_Z_SUPPORT=1 -DBXZSTR_BZ2_SUPPORT=0 -DBXZSTR_LZMA_SUPPORT=0 -DBXZSTR_ZSTD_SUPPORT=0)
O="$OUT/obj"
for f in krakenutil seqreader hyperloglogplus; do
  if [ ! -f "$O/$f.o" ] || [ "$SRC/$f.cpp" -nt "$O/$f.o" ]; then "$CXX" "${CXXFLAGS[@]}" -c "$SRC/$f.cpp" -o "$O/$f.o"; fi
done
"$CXX" "${CXXFLAGS[@]}" -o "$OUT/count_unique" "$SRC/count_unique.cpp" $O/krakenutil.o $O/seqreader.o $O/hyperloglogplus.o -lz
echo "oracle/_ref/count_unique built"
