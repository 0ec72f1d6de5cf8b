#!/bin/bash
# Build a tuning variant of the direct-J/K class kernels into pyscf_b200/libb200jk_<name>.so (git-ignored, travels to the
# GPU box): the 10 bra-class translation units are recompiled with extra nvcc flags (and, optionally, with header files
# taken from another git revision), everything else is linked from the regular build.
# usage: tools/build_variant.sh <name> "<extra nvcc flags>" [<git rev> <file> ...]
set -e
NAME=$1; FLAGS=$2; shift 2
ROOT=$(cd "$(dirname "$0")/.." && pwd)
SRC=/tmp/b200jk_variant_$NAME
rm -rf $SRC; mkdir -p $SRC/csrc $SRC/include $SRC/obj
cp $ROOT/pyscf_b200/csrc/*.cu $ROOT/pyscf_b200/csrc/*.cuh $ROOT/pyscf_b200/csrc/*.hpp $SRC/csrc/
cp $ROOT/include/b200jk.h $SRC/include/
mkdir -p $SRC/csrc/../../include && cp $ROOT/include/b200jk.h $SRC/csrc/../../include/ 2>/dev/null || true
if [ $# -gt 1 ]; then REV=$1; shift; for f in "$@"; do git -C $ROOT show $REV:pyscf_b200/csrc/$f > $SRC/csrc/$f; done; fi
NV="nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC -Xptxas -v -I$ROOT/include $FLAGS"
cd $SRC/csrc
for i in 0 1 2 3 4 5 6 7 8 9; do
  ( $NV -DB2_BRA_ID=$i -c jk_class_tu.cu -o $SRC/obj/jk_bra_$i.o 2> $SRC/obj/ptxas_$i.log || { cat $SRC/obj/ptxas_$i.log; exit 1; } ) &
  if (( i % 4 == 3 )); then wait; fi
done
wait
B=$ROOT/pyscf_b200/csrc/build
nvcc -shared -o $ROOT/pyscf_b200/libb200jk_$NAME.so $B/b200jk.o $SRC/obj/jk_bra_*.o $B/df.o $B/i8gemm.o $B/df_lk_*.o $B/rys_blob.o -lcublas -lcusolver -lcudart 2>/dev/null
ls -la $ROOT/pyscf_b200/libb200jk_$NAME.so
grep -h "spill stores" $SRC/obj/ptxas_*.log | grep -vc " 0 bytes spill stores" || true
