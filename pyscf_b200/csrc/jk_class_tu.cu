// jk_class_tu.cu — compiled once per bra pair class (-DB2_BRA_ID=0..9): instantiates the kernels
// (bra class | every ket class <= bra class).  With B200JK_EMULATE and no B2_BRA_ID: all classes.
#ifndef B200JK_EMULATE
#include <cuda_runtime.h>
#endif
#include <string>
#include "jk_classes.cuh"

namespace b200jk {
#define X(id, li, lj) \
    void launch_bra_##id(int ck, const KParams& P, b2_stream_t st) { launch_ket<li, lj>(ck, P, st); } \
    void info_bra_##id(int ck, int* out) { info_ket<li, lj>(ck, out); }
#if !defined(B2_BRA_ID)
B2_PAIR_CASES(X)
#elif B2_BRA_ID == 0
X(0, 0, 0)
#elif B2_BRA_ID == 1
X(1, 1, 0)
#elif B2_BRA_ID == 2
X(2, 1, 1)
#elif B2_BRA_ID == 3
X(3, 2, 0)
#elif B2_BRA_ID == 4
X(4, 2, 1)
#elif B2_BRA_ID == 5
X(5, 2, 2)
#elif B2_BRA_ID == 6
X(6, 3, 0)
#elif B2_BRA_ID == 7
X(7, 3, 1)
#elif B2_BRA_ID == 8
X(8, 3, 2)
#elif B2_BRA_ID == 9
X(9, 3, 3)
#endif
#undef X
}  // namespace b200jk
