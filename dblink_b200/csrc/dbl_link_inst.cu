// One translation unit per attribute count: compiled with -DDBL_INST_A=<A>; instantiates k_link_pcg2<A, 0..A, ...>.
#include "dbl_link_pcg2.cuh"

#ifndef DBL_INST_A
#error "compile with -DDBL_INST_A=<number of attributes>"
#endif

#define DBL_CAT2(a, b) a##b
#define DBL_CAT(a, b) DBL_CAT2(a, b)

Pcg2Kernel DBL_CAT(dbl_pcg2_kernel_a, DBL_INST_A)(int ns, Pcg2Format f) {
  return pcg2_kernel<DBL_INST_A, DBL_INST_A>(ns, f);
}
