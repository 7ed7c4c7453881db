#!/bin/bash
# Experiment build of the library: tools/build_variant.sh NAME [-DFLAG ...]  ->  lab/NAME.so (git-ignored, travels to
# the GPU machine).  Used with PG_LIB_VARIANT=NAME tools/prof_edge.py / tools/prof_pool.py / tools/prof_graph.py.
# The Makefile's own recipe and sources, with the flags appended, into build/var_NAME; always rebuilt (-B), since
# the flags of an earlier build of the same NAME may differ.
set -e
name=$1; shift
csrc="$(dirname "$0")/../point-gnn_b200/csrc"
make -B -C "$csrc" -j "$(nproc)" BUILD="build/var_$name" OUT="../../lab/$name.so" EXTRA_NVCCFLAGS="$*"
grep -A3 "wg_gemm_kernel" "$csrc/build/var_$name/pg_tc.ptxas.log" | grep -E "registers|spill"
