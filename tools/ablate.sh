#!/bin/bash
# builds variants of the library for timing experiments:  tools/ablate.sh name1:"-DFOO -DBAR=1" name2:"..."
set -e
cd "$(dirname "$0")/../elprep_b200/csrc"
mkdir -p ../lib/exp
rm -f ../lib/exp/*.so
SRCS="api.cu bgzf.cpp bam_ingest.cu sort.cu markdup.cu optical.cu coordsort.cu bqsr_gather.cu bqsr_apply.cu bqsr_finalize.cu"
FL="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC,-ffp-contract=off -shared"
for spec in "$@"; do
  name="${spec%%:*}"; defs="${spec#*:}"; [ "$defs" = "$spec" ] && defs=""
  nvcc $FL $defs -o ../lib/exp/lib_$name.so $SRCS -lcudart -lz &
done
wait
ls ../lib/exp
