#!/bin/bash
# Experiment build of the library: tools/build_variant.sh NAME [-DFLAG ...]  ->  lab/NAME.so (git-ignored, travels to
# the GPU machine).  Used with PG_LIB_VARIANT=NAME tools/prof_pool.py / tools/prof_graph.py.
set -e
name=$1; shift
cd "$(dirname "$0")/../point-gnn_b200/csrc"
mkdir -p build/var_$name ../../lab
for f in pg_api pg_graph pg_ops pg_edge_simt pg_tc pg_post pg_input; do
  /usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC \
    -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr -Xptxas -v "$@" -c $f.cu -o build/var_$name/$f.o \
    2> build/var_$name/$f.ptxas.log &
done
wait
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../lab/$name.so build/var_$name/*.o -lcudart
grep -A3 "wg_gemm_kernel" build/var_$name/pg_tc.ptxas.log | grep -E "registers|spill"
