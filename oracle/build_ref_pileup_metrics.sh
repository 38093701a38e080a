#!/usr/bin/env bash
# oracle/build_ref_pileup_metrics.sh -- TEST INFRASTRUCTURE, not product code.
#
# Links oracle/ref_harness_pileup_metrics.cpp against the reference archives oracle/build_ref.sh leaves in oracle/_ref/build (the
# UNMODIFIED reference sources, with the same flags) into oracle/_ref/libstrelka_ref_pileup_metrics.so.  Run it after build_ref.sh.
set -euo pipefail

HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${STRELKA_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
B="$OUT/build"

if [[ ! -d "$REF/src/c++/lib" || ! -f "$B/libapp_starling.a" ]]; then
    echo "build_ref_pileup_metrics.sh: reference tree or oracle/_ref/build archives not found (using prebuilt oracle/_ref if present)" >&2
    exit 0
fi

INC="-I$B/gen -I$REF/src/c++/lib -I$B/boost_1_58_0_subset -I$B/htslib-1.7-6-g6d2bfb7 -I$B/rapidjson-1.1.0/include -I$B/CodeMin-1.0.5/include"
CXXFLAGS="-std=c++11 -O3 -fomit-frame-pointer -fPIC -w"
g++ $CXXFLAGS $INC -include limits -c "$HERE/ref_harness_pileup_metrics.cpp" -o "$B/obj/ref_harness_pileup_metrics.o"
g++ -shared -o "$OUT/libstrelka_ref_pileup_metrics.so" "$B/obj/ref_harness_pileup_metrics.o" \
    -Wl,--start-group "$B/libapp_starling.a" "$B/libcommon.a" -Wl,--end-group "$B/libboost.a" "$B/htslib-1.7-6-g6d2bfb7/libhts.a" -lz -lpthread
echo "built $OUT/libstrelka_ref_pileup_metrics.so"
