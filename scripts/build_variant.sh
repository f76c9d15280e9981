#!/bin/bash
# Builds deodr_b200/libdeodr_b200_<name>.so with extra nvcc flags (A/B experiments: DEODR_B200_LIB selects it at run time).
#   scripts/build_variant.sh tilez4 -DDEODR_TILEZ_MIN_CTAS=4
#   scripts/build_variant.sh exact -DDEODR_EXACT_SHORT_WRAP=1
# The translation units are those of __graft_entry__.UNITS, so that a variant exports every symbol _cabi.load() binds.
name=$1; shift
cd "$(dirname "$0")/.."
units=$(python -c 'import __graft_entry__ as e; print(" ".join(e.UNITS))') || exit 1
mkdir -p build_$name
pids=()
objs=()
for u in $units; do
  "${NVCC:-/usr/local/cuda/bin/nvcc}" -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-pthread "$@" \
     -c -o build_$name/${u%.*}.o deodr_b200/csrc/$u &
  pids+=($!)
  objs+=(build_$name/${u%.*}.o)
done
for p in "${pids[@]}"; do wait $p || exit 1; done
"${NVCC:-/usr/local/cuda/bin/nvcc}" -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fPIC,-pthread -o deodr_b200/libdeodr_b200_$name.so "${objs[@]}"
ls -la deodr_b200/libdeodr_b200_$name.so
