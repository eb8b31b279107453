#!/bin/bash
# builds variants of the library for timing experiments:  tools/ablate.sh name1:"-DFOO -DBAR=1" name2:"..."
# -> elprep_b200/lib/exp/lib_<name>.so.  Every source but bqsr_gather.cu is compiled once (tools/_build/ablate/); the defines apply
# to bqsr_gather.cu, which holds the BQSR gather kernels (the CNT_ABL_* switches of bqsr_count.inl).
set -e
CSRC="$(cd "$(dirname "$0")/../elprep_b200/csrc" && pwd)"
OBJ="$(cd "$(dirname "$0")" && pwd)/_build/ablate"
cd "$CSRC"
rm -rf "$OBJ"; mkdir -p ../lib/exp "$OBJ"
rm -f ../lib/exp/*.so
SRCS=$(make -s -n -p 2>/dev/null | awk -F' = ' '$1 == "SRCS" { print $2; exit }')
NOFMA_SRCS=$(make -s -n -p 2>/dev/null | awk -F' = ' '$1 == "NOFMA_SRCS" { print $2; exit }')
FL="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC,-ffp-contract=off"
for s in $SRCS $NOFMA_SRCS; do
  [ "$s" = bqsr_gather.cu ] && continue
  extra=""; case " $NOFMA_SRCS " in *" $s "*) extra="-fmad=false";; esac
  o="$OBJ/${s%.*}.o"
  nvcc $FL $extra -c -o "$o" "$s" &
done
wait
for spec in "$@"; do
  name="${spec%%:*}"; defs="${spec#*:}"; [ "$defs" = "$spec" ] && defs=""
  nvcc $FL $defs -c -o "$OBJ/bqsr_gather_$name.o" bqsr_gather.cu
  nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../lib/exp/lib_$name.so $(ls "$OBJ"/*.o | grep -v '/bqsr_gather_') "$OBJ/bqsr_gather_$name.o" -lcudart -lz -ldl
done
ls ../lib/exp
