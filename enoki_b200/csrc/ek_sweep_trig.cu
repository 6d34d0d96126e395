/*
 * ek_sweep_trig.cu -- the instantiations of the general sweep kernel (ek_sweep.cu) that carry tan / cot / asin / acos /
 * atan / atan2, sinh / cosh / tanh / asinh / acosh / atanh / cbrt, erf / erfc / erfinv / lgamma / tgamma, pow /
 * frexp / hypot / dawson / erfi and carlson_rf / carlson_rd / carlson_rc (ek_sweep_kernel<V, INLINE, true>).  They are compiled here, into a module of their own, so that ek_sweep.o
 * holds exactly the kernels every other program runs, laid out as they were before these operations existed.
 */
#define EK_SWEEP_TRIG_TU
#include "ek_sweep.cu"
