/*
 * ek_sweep_fast_trig.cu -- the instantiations of the 32-bit fast sweep kernel (ek_sweep_fast.cu) that carry tan / cot /
 * asin / acos / atan / atan2 (ek_fast_kernel<T, EK_FX_TRIG>, <T, EK_FX_F16 | EK_FX_TRIG>) or sinh / cosh / tanh / asinh /
 * acosh / atanh / cbrt (<T, EK_FX_HYP>, and <T, EK_FX_F16 | EK_FX_TRIG | EK_FX_HYP> for a body that mixes them with the
 * first two sets) or erf / erfc / erfinv / lgamma / tgamma (<T, EK_FX_SPEC>, and <T, EK_FX_ALL & ~EK_FX_MATH> for a body
 * that mixes them with the first three sets) or pow / frexp / hypot / dawson / erfi (<T, EK_FX_MATH>, and
 * <T, EK_FX_ALL & ~EK_FX_ELL> for a body that mixes them with the first four sets) or carlson_rf / carlson_rd /
 * carlson_rc (<T, EK_FX_ELL>, and <T, EK_FX_ALL> for a body that mixes them with anything else).  They are compiled
 * here, into a module
 * of their own, so that ek_sweep_fast.o holds exactly the kernels every other program runs, laid out as they were before
 * these operations existed.
 */
#define EK_FAST_TRIG_TU
#include "ek_sweep_fast.cu"
