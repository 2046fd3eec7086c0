// TEST INFRASTRUCTURE ONLY.  C-linkage shim around the reference's own ODE Dantzig solver so tests can call it
// through ctypes.  Compiled together with the sources under <REF>/dart/external/odelcpsolver/ (never
// copied) into oracle/_ref/libodelcp.so by oracle/Makefile.
//   reference: dart/external/odelcpsolver/lcp.h:60 (dSolveLCP), common.h:141 (dPAD)
#include "dart/external/odelcpsolver/lcp.h"
#include "dart/external/odelcpsolver/common.h"

extern "C" {
int ref_dPAD(int n) { return dPAD(n); }
// A: n x dPAD(n) row-major (clobbered), x/w out, b/lo/hi clobbered.  Returns 1 on success.
int ref_dSolveLCP(int n, double* A, double* x, double* b, double* w, int nub, double* lo, double* hi, int* findex,
                  int earlyTermination) {
  return dSolveLCP(n, A, x, b, w, nub, lo, hi, findex, earlyTermination != 0) ? 1 : 0;
}
}
